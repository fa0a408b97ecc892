#!/usr/bin/env python
"""The reward and target step of training (dataloader.py populate_buffer after load_gz_log_files) on arena logs, in the trainer's
file batches: (a) the reference's path restated — a CPU float64 GRP over every prefix list per Gameplay (reward_calculator.py)
plus the per-move Python loop (steps_to_done, player ranks, the buffer entries) — against (b) mortal_b200.reward.training_samples
(k_grp_matrix once per game, k_train_targets). Both paths end in a device synchronise and are checked equal (targets exactly,
rewards within 1e-10). Also k_grp_matrix alone over all games' rows, device-resident (CUDA events after warm-up). The GRP has the
default shape (hidden 64, 2 layers) with random weights; the logs are produced on the spot by the arena. Prints the GPU name and
power limit beside the numbers. Not part of the pytest suite."""
import argparse
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import reward_lib as R
from mortal_b200 import _lib
from mortal_b200.dataset import GameplayLoader
from mortal_b200.libriichi.arena import OneVsThree
from mortal_b200.reward import RewardCalculator, training_samples

ap = argparse.ArgumentParser()
ap.add_argument("--games", type=int, default=1024, help="arena games (a multiple of 4)")
ap.add_argument("--batch", type=int, default=20, help="files per batch (the trainer's file_batch_size)")
ap.add_argument("--reps", type=int, default=50, help="timed k_grp_matrix launches")
args = ap.parse_args()


class Eng:
    engine_type, version, is_oracle, enable_quick_eval, enable_rule_based_agari_guard = "mortal", 4, False, True, False

    def __init__(self, name, bias):
        self.name, self.bias = name, bias

    def react_device(self, obs, masks):
        q = torch.rand(masks.shape, device=masks.device)
        q[:, :34] += self.bias * obs[:, 876, :] + obs[:, 875, :]
        q = q.masked_fill(~masks, -1.0)
        return q.argmax(-1), q


def reference_path(data, net, pts):
    """populate_buffer restated: per Gameplay the CPU GRP and the per-move loop; -> (buffer, steps, rewards, ranks)"""
    buffer, cols = [], ([], [], [])
    for file in data:
        for game in file:
            obs, actions, masks = game.take_obs(), game.take_actions(), game.take_masks()
            at_kyoku, dones, apply_gamma = game.take_at_kyoku(), game.take_dones(), game.take_apply_gamma()
            if not at_kyoku:
                continue
            grp, player_id = game.take_grp(), game.take_player_id()
            kyoku_rewards = R.ref_delta_pt(R.ref_calc_grp(net, grp.take_feature()), pts, False, player_id, grp.take_rank_by_player())
            steps, rewards, ranks = R.ref_targets(kyoku_rewards, player_id, grp.take_feature(), grp.take_final_scores(), at_kyoku,
                                                  dones, apply_gamma)
            for i in range(len(at_kyoku)):
                buffer.append([obs[i], actions[i], masks[i], steps[i], rewards[i], ranks[i]])
            for c, v in zip(cols, (steps, rewards, ranks)):
                c.append(v)
    torch.cuda.synchronize()
    return buffer, *(np.concatenate(c) for c in cols)


gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
torch.manual_seed(0)
net = R.random_grp(64, 2, 1)
pts = [90, 45, 0, -135]
rc = RewardCalculator(net, pts)
with tempfile.TemporaryDirectory() as d:
    OneVsThree(disable_progress_bar=True, log_dir=d).py_vs_py(Eng("alpha", 2.0), Eng("beta", 0.5), (95000, 41), args.games // 4)
    files = sorted(os.path.join(d, f) for f in os.listdir(d))
    loader = GameplayLoader(4, oracle=False)
    t_ref = t_dev = 0.0
    n_samples = n_gameplays = 0
    err = 0.0
    feats = []
    for b in range(0, len(files), args.batch):
        data = loader.load_gz_log_files(files[b:b + args.batch])
        torch.cuda.synchronize()
        if b == 0:  # warm-up of both paths on the first batch
            reference_path(data, net, pts)
            training_samples(data, rc)
            torch.cuda.synchronize()
        t0 = time.perf_counter()
        _, ws, wr, wk = reference_path(data, net, pts)
        t1 = time.perf_counter()
        got = training_samples(data, rc)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        t_ref += t1 - t0
        t_dev += t2 - t1
        assert np.array_equal(got["steps_to_done"].cpu().numpy(), ws) and np.array_equal(got["player_ranks"].cpu().numpy(), wk)
        err = max(err, float(np.abs(got["kyoku_rewards"].cpu().numpy() - wr).max()))
        n_samples += len(ws)
        n_gameplays += sum(len(f) for f in data)
        feats += [f[0].take_grp().take_feature() for f in data if f]
        del data, got
assert err <= 1e-10

# k_grp_matrix alone: every game's rows resident on the device, no jobs
L = _lib.load()
dev = torch.device("cuda", 0)
off = np.zeros(len(feats) + 1, dtype=np.int32)
np.cumsum([len(f) for f in feats], out=off[1:])
feat_d = torch.from_numpy(np.concatenate(feats)).to(dev)
off_d = torch.from_numpy(off).to(dev)
matrix = torch.empty((int(off[-1]), 4, 4), dtype=torch.float64, device=dev)
stream = torch.cuda.current_stream(dev)


def launch():
    _lib.check(L.mjx_grp_reward_dev(len(feats), feat_d.data_ptr(), off_d.data_ptr(), int(off[-1]), rc.weights.data_ptr(),
                                    rc.weights.numel(), rc.hidden, rc.layers, matrix.data_ptr(), 0, None, 0, None, None, None, None,
                                    None, None, None, rc._pts_host, 0, None, None, None, None, stream.cuda_stream), "mjx_grp_reward_dev")


for _ in range(5):
    launch()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(stream)
for _ in range(args.reps):
    launch()
e1.record(stream)
torch.cuda.synchronize()
k_ms = e0.elapsed_time(e1) / args.reps
ref_m = torch.cat([R.ref_calc_grp(net, f) for f in feats[:32]])
assert (matrix[:len(ref_m)].cpu() - ref_m).abs().max().item() <= 1e-12

n_batches = (len(files) + args.batch - 1) // args.batch
print(f"GPU: {gpu}")
print(f"{len(files)} files in {n_batches} batches of {args.batch}: {n_gameplays} Gameplays, {n_samples} samples, "
      f"{int(off[-1])} kyoku rows in {len(feats)} games")
print(f"(a) reference path (CPU GRP per Gameplay + per-move loop): {t_ref:.3f} s total, {1e3 * t_ref / n_batches:.2f} ms per batch")
print(f"(b) training_samples:                                      {t_dev:.3f} s total, {1e3 * t_dev / n_batches:.2f} ms per batch "
      f"({t_ref / t_dev:.1f}x)")
print(f"k_grp_matrix alone, {len(feats)} games / {int(off[-1])} rows, device-resident: {k_ms:.3f} ms per launch")
print(f"agreement: steps_to_done and player_ranks equal, max |kyoku reward (a) - (b)| = {err:.3e}")
