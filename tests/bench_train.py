#!/usr/bin/env python
"""Policy-net training throughput: the reference's train_batch restated against the fused path (not part of the pytest suite).

    python tests/bench_train.py [--games 16] [--steps 20] [--warmup 5] [--rounds 5] [--batches 8]

Generates arena logs on the spot (`--games` sets of 4 hanchan), loads `--batches` batches of 512 through the device
FileDatasetsIter, then, for float32 and for float16 AMP (torch.autocast + GradScaler), trains a version-4 192 x 40 Brain + DQN +
AuxNet from the same initial weights in two arms, alternated window by window in one process:
  (a) mortal/train.py's train_batch: Brain.forward + DQN + AuxNet + the torch loss expressions, backward, AdamW;
  (b) Brain.forward_train + DQN.heads + AuxNet + train_ops.dqn_losses, backward, the same AdamW.
Each window is `--steps` steps after `--warmup`, ending in a device synchronise. It prints the median steps/s per arm over the
`--rounds` windows (and every window's), each arm's device time per step and the fused kernels' share of it (torch.profiler over
3 steps; kernels of csrc/mjx_train.cuh), the largest per-step relative loss difference between the arms over the first window,
and the GPU's name and power limit read in the same run, as one JSON line."""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch
from torch.nn import functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from mortal_b200 import train_ops  # noqa: E402
from mortal_b200.dataloader import FileDatasetsIter  # noqa: E402
from mortal_b200.libriichi.arena import OneVsThree  # noqa: E402
from mortal_b200.model import DQN, GRP, AuxNet, Brain  # noqa: E402
from test_gpu_gameplay_decode import _Eng  # noqa: E402

GAMMA, MIN_Q, NEXT_RANK, BATCH = 1.0, 5.0, 0.2, 512


def reference_step(brain, dqn, aux, bt):
    obs, actions, masks, steps_to_done, rewards, ranks = bt
    q_target = (GAMMA ** steps_to_done * rewards).to(torch.float32)
    phi = brain(obs)
    q_out = dqn(phi, masks)
    q = q_out[range(BATCH), actions]
    dqn_loss = 0.5 * F.mse_loss(q, q_target)
    cql_loss = q_out.logsumexp(-1).mean() - q.mean()
    nr_loss = F.cross_entropy(aux(phi)[0], ranks)
    return dqn_loss + cql_loss * MIN_Q + nr_loss * NEXT_RANK


def fused_step(brain, dqn, aux, bt):
    obs, actions, masks, steps_to_done, rewards, ranks = bt
    phi = brain.forward_train(obs)
    v, a = dqn.heads(phi)
    dqn_loss, cql_loss, nr_loss, *_ = train_ops.dqn_losses(v, a, aux(phi)[0], masks, actions, steps_to_done, rewards, ranks, GAMMA)
    return dqn_loss + cql_loss * MIN_Q + nr_loss * NEXT_RANK


class Arm:
    def __init__(self, models, step_fn, amp):
        self.models = [copy.deepcopy(m).train() for m in models]
        self.step_fn, self.amp = step_fn, amp
        self.opt = torch.optim.AdamW([p for m in self.models for p in m.parameters()], lr=1e-5)
        self.scaler = torch.amp.GradScaler("cuda", enabled=amp)

    def step(self, bt):
        with torch.autocast("cuda", enabled=self.amp):
            loss = self.step_fn(*self.models, bt)
        self.scaler.scale(loss).backward()
        self.scaler.step(self.opt)
        self.scaler.update()
        self.opt.zero_grad(set_to_none=True)
        return loss.detach()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, default=16)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batches", type=int, default=8)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    torch.backends.cudnn.benchmark = True
    with tempfile.TemporaryDirectory() as d:
        torch.manual_seed(0)
        OneVsThree(disable_progress_bar=True, log_dir=d).py_vs_py(_Eng("alpha", 2.0), _Eng("beta", 0.5), (99000, 7), args.games)
        files = sorted(os.path.join(d, f) for f in os.listdir(d))
        batches = []
        for bt in FileDatasetsIter(4, files, [6.0, 4.0, 2.0, 0.0], file_batch_size=len(files), grp=GRP(), batch_size=BATCH):
            if bt[0].shape[0] == BATCH:
                batches.append(bt)
            if len(batches) == args.batches:
                break
    torch.manual_seed(1)
    models = (Brain(conv_channels=192, num_blocks=40, version=4).cuda(), DQN(version=4).cuda(), AuxNet((4,)).cuda())
    result = {"gpu": gpu[0] if gpu else torch.cuda.get_device_name(), "batch": BATCH, "brain": "v4 192x40", "n_batches": len(batches)}
    for name, amp in (("fp32", False), ("fp16_amp", True)):
        ref, fus = Arm(models, reference_step, amp), Arm(models, fused_step, amp)
        # loss agreement over the first window, from the same weights on the same batches
        diffs = []
        for i in range(args.steps):
            lr_, lf = ref.step(batches[i % len(batches)]), fus.step(batches[i % len(batches)])
            diffs.append(abs(lf.item() - lr_.item()) / abs(lr_.item()))
        times = {"reference": [], "fused": []}
        for _ in range(args.rounds):
            for arm_name, arm in (("reference", ref), ("fused", fus)):
                for i in range(args.warmup):
                    arm.step(batches[i % len(batches)])
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for i in range(args.steps):
                    arm.step(batches[i % len(batches)])
                torch.cuda.synchronize()
                times[arm_name].append(args.steps / (time.perf_counter() - t0))
        device_ms = {}
        for arm_name, arm in (("reference", ref), ("fused", fus)):
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for i in range(3):
                    arm.step(batches[i % len(batches)])
                torch.cuda.synchronize()
            events = prof.key_averages()
            device_ms[arm_name] = sum(e.self_device_time_total for e in events) / 3e3
            if arm is fus:
                device_ms["fused_kernels"] = sum(e.self_device_time_total for e in events if "mjx_train" in e.key) / 3e3
        med = {k: statistics.median(v) for k, v in times.items()}
        result[name] = {"reference_steps_per_s": med["reference"], "fused_steps_per_s": med["fused"], "speedup": med["fused"] / med["reference"],
                        "reference_all": times["reference"], "fused_all": times["fused"],
                        "reference_device_ms_per_step": device_ms["reference"], "fused_device_ms_per_step": device_ms["fused"],
                        "fused_kernels_ms_per_step": device_ms["fused_kernels"], "max_rel_loss_diff": max(diffs),
                        "first_rel_loss_diff": diffs[0]}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
