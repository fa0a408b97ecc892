#!/usr/bin/env python
"""Data-parallel policy-net training throughput (not part of the pytest suite).

    python tests/bench_train_ddp.py [--games 16] [--steps 20] [--warmup 5] [--rounds 3] [--batches 8] [--amp]

Generates arena logs on the spot (`--games` sets of 4 hanchan), then for every rank count W = 1 .. (GPUs present) and for the
global batches 512 and W x 512 runs mortal_b200.train's `_Trainer.step` (version-4 192 x 40 Brain, synchronised BatchNorm, one
gradient all-reduce per step, AdamW, GradScaler) on W ranks over NCCL, one per GPU (W = 1: one process, no process group). Each
rank trains on its contiguous shard of the logs (the trainer's shard rule) at batch / W. A window is `--steps` steps after
`--warmup`, ending in a device synchronise and a barrier; the median over `--rounds` windows gives steps/s and samples/s. A
separate torch.profiler run over 3 steps gives rank 0's device time per step and the NCCL kernel time in it, split into the
gradient all-reduce (the longest NCCL kernel of each step) and the rest (the 162 BatchNorm exchanges of the 81 training-mode
BatchNorms). The GPU's name and power limit are read in the same run. Prints one JSON line."""
import argparse
import json
import os
import socket
import statistics
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def config(d, batch, amp):
    from mortal_b200.model import DQN, Brain, mortal_state_dict

    torch.manual_seed(1)
    b = Brain(conv_channels=32, num_blocks=2, version=4)
    torch.save({"mortal": mortal_state_dict(b), "current_dqn": DQN(version=4).state_dict(),
                "config": {"control": {"version": 4}, "resnet": {"conv_channels": 32, "num_blocks": 2}}}, os.path.join(d, "base.pth"))
    return {
        "control": {"version": 4, "online": False, "batch_size": batch, "opt_step_every": 1, "save_every": 1000, "test_every": 1000,
                    "device": "cuda:0", "enable_cudnn_benchmark": True, "enable_amp": amp, "enable_compile": False,
                    "state_file": os.path.join(d, "mortal.pth"), "best_state_file": os.path.join(d, "best.pth")},
        "env": {"gamma": 1.0, "pts": [6.0, 4.0, 2.0, 0.0]},
        "resnet": {"conv_channels": 192, "num_blocks": 40},
        "cql": {"min_q_weight": 5.0}, "aux": {"next_rank_weight": 0.2}, "freeze_bn": {"mortal": False},
        "optim": {"eps": 1e-8, "betas": [0.9, 0.999], "weight_decay": 0.1, "max_grad_norm": 1.0,
                  "scheduler": {"peak": 1e-4, "final": 1e-5, "warm_up_steps": 10, "max_steps": 100000}},
        "test_play": {"games": 4, "log_dir": os.path.join(d, "test_play")},
        "baseline": {"test": {"device": "cuda:0", "state_file": os.path.join(d, "base.pth")}},
    }


def worker(args):
    """one rank: time `_Trainer.step` and profile it, write rank 0's findings to args.out"""
    import torch.distributed as dist

    from mortal_b200.dataloader import FileDatasetsIter
    from mortal_b200.model import GRP
    from mortal_b200.train import _Trainer, shard

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    device = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(device)
    if world > 1:
        dist.init_process_group("nccl", device_id=device)
    d = tempfile.mkdtemp()
    cfg = config(d, args.batch, args.amp)
    cfg["control"]["device"] = cfg["baseline"]["test"]["device"] = str(device)
    T = _Trainer(cfg, online=False)
    files = sorted(os.path.join(args.logs, f) for f in os.listdir(args.logs))
    batches = []
    for bt in FileDatasetsIter(4, shard(files, rank, world), cfg["env"]["pts"], file_batch_size=len(files), grp=GRP(),
                               batch_size=T.batch_size, device=device.index):
        if bt[0].shape[0] == T.batch_size:
            batches.append(bt)
        if len(batches) == args.batches:
            break
    assert len(batches) == args.batches, f"rank {rank}: only {len(batches)} batches of {T.batch_size} in its shard"

    def window(n):
        for i in range(n):
            T.step(*batches[i % len(batches)])
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()

    rates = []
    for _ in range(args.rounds):
        window(args.warmup)
        t0 = time.perf_counter()
        window(args.steps)
        rates.append(args.steps / (time.perf_counter() - t0))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        window(3)
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    nccl = sorted((e.device_time for e in kernels if "nccl" in e.name.lower()), reverse=True)
    grad_us = sum(nccl[:3]) if nccl else 0.0
    if rank == 0:
        med = statistics.median(rates)
        with open(args.out, "w") as f:
            json.dump({"world": world, "global_batch": args.batch, "amp": args.amp, "steps_per_s": med, "samples_per_s": med * args.batch,
                       "steps_per_s_all": rates, "device_ms_per_step": sum(e.device_time for e in kernels) / 3e3,
                       "nccl_kernels_per_step": len(nccl) / 3, "grad_allreduce_ms_per_step": grad_us / 3e3,
                       "bn_exchange_ms_per_step": (sum(nccl) - grad_us) / 3e3}, f)
    if world > 1:
        dist.destroy_process_group()


def free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, default=16)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--amp", action="store_true")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--batch", type=int, default=512, help=argparse.SUPPRESS)
    ap.add_argument("--logs", help=argparse.SUPPRESS)
    ap.add_argument("--out", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    from mortal_b200.libriichi.arena import OneVsThree
    from test_gpu_gameplay_decode import _Eng

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    n_gpus = torch.cuda.device_count()
    if n_gpus < 1:
        raise SystemExit("bench_train_ddp: no CUDA device")
    runs = []
    with tempfile.TemporaryDirectory() as d:
        logs = os.path.join(d, "logs")
        torch.manual_seed(0)
        OneVsThree(disable_progress_bar=True, log_dir=logs).py_vs_py(_Eng("alpha", 2.0), _Eng("beta", 0.5), (99000, 7), args.games)
        for world in range(1, n_gpus + 1):
            for batch in sorted({512, 512 * world}):
                out = os.path.join(d, f"w{world}_b{batch}.json")
                cmd = [os.path.abspath(__file__), "--worker", "--batch", str(batch), "--logs", logs, "--out", out,
                       "--steps", str(args.steps), "--warmup", str(args.warmup), "--rounds", str(args.rounds),
                       "--batches", str(args.batches)] + (["--amp"] if args.amp else [])
                if world > 1:
                    cmd = ["-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
                           "--master-port", str(free_port())] + cmd
                subprocess.run([sys.executable] + cmd, check=True, env=dict(os.environ, OMP_NUM_THREADS="1"))
                with open(out) as f:
                    runs.append(json.load(f))
    print(json.dumps({"gpu": gpu, "n_gpus": n_gpus, "brain": "v4 192x40", "runs": runs}))


if __name__ == "__main__":
    main()
