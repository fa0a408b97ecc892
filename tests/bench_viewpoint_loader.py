#!/usr/bin/env python
"""GameplayLoader(4, oracle=False).load_gz_log_files on single-viewpoint logs against the full logs of the same players: every arena
log is written once with distinct seat names (full) and once as each seat sees it (the other seats' haipai and draws "?"); batches
of the same files and player are loaded masked and full alternately, outputs checked equal, and a call is split into read + gunzip,
decode and replay + encode. A masked log replays from the player's own seat (one seat's per-event work instead of four), so replay +
encode is the figure to compare. Also: how many masked logs the device decoder declined, and k_replay_viewpoints alone (CUDA events
over --reps launches after warm-up) on the jobs of all masked logs. Logs are produced on the spot by the arena, so the tool needs no
dataset. Prints the GPU name and power limit beside the numbers."""
import argparse
import gzip
import json
import multiprocessing
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

from mortal_b200 import _lib, _logio
from mortal_b200.dataset import GameplayLoader
from mortal_b200.env import ReplayEnv
from mortal_b200.libriichi.arena import OneVsThree
from mortal_b200.validate_logs import decode_dev
from viewpoint_lib import named, viewpoint

ap = argparse.ArgumentParser()
ap.add_argument("--games", type=int, default=1024, help="arena games (a multiple of 4)")
ap.add_argument("--batch", type=int, default=80, help="files per load_gz_log_files call (one player each)")
ap.add_argument("--batches", type=int, default=8, help="loader calls timed per kind")
ap.add_argument("--reps", type=int, default=20, help="timed kernel launches")
args = ap.parse_args()


def write(path, events):
    with gzip.open(path, "wt") as f:
        f.write("".join(json.dumps(ev) + "\n" for ev in events))


def write_copies(job):
    """one arena log -> its full copy (distinct seat names) and the four masked copies"""
    fn, full, masked = job
    with gzip.open(fn, "rt") as f:
        ev = [json.loads(ln) for ln in f if ln.strip()]
    write(full, named(ev))
    for p in range(4):
        write(masked[p], viewpoint(ev, p))


# the copies are written by worker processes, forked here before CUDA is initialised in this process
pool = multiprocessing.get_context("fork").Pool(min(32, os.cpu_count() or 1))


class Eng:
    engine_type, version, is_oracle, enable_quick_eval, enable_rule_based_agari_guard = "mortal", 4, False, True, False

    def __init__(self, name):
        self.name = name

    def react_device(self, obs, masks):
        q = torch.rand(masks.shape, device=masks.device)
        q[:, :34] += 2.0 * obs[:, 876, :] + obs[:, 875, :]
        q = q.masked_fill(~masks, -1.0)
        return q.argmax(-1), q


T = {}
_orig_device, _orig_replay = GameplayLoader._load_device, GameplayLoader._replay


def _timed_device(self, logs):
    t0 = time.perf_counter()
    try:
        return _orig_device(self, logs)
    finally:
        torch.cuda.synchronize()
        T["load"] = time.perf_counter() - t0


def _timed_replay(self, jobs, firsts, grps):
    t0 = time.perf_counter()
    r = _orig_replay(self, jobs, firsts, grps)
    torch.cuda.synchronize()
    T["replay"] = time.perf_counter() - t0
    return r


GameplayLoader._load_device, GameplayLoader._replay = _timed_device, _timed_replay


def load(files, p):
    """one loader call for seat p -> (result, {stage: seconds})"""
    T.clear()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = GameplayLoader(4, oracle=False, player_names=[f"challenger.{p}", f"champion.{p}"]).load_gz_log_files(files)
    torch.cuda.synchronize()
    total = time.perf_counter() - t0
    return r, {"read + gunzip": total - T["load"], "decode": T["load"] - T["replay"], "replay + encode": T["replay"], "total": total}


def same(a, b):
    for pa, pb in zip(a, b, strict=True):
        for x, y in zip(pa, pb, strict=True):
            assert x.take_player_id() == y.take_player_id() and x.player_name == y.player_name
            assert torch.equal(x.take_obs(), y.take_obs()) and torch.equal(x.take_masks(), y.take_masks())
            assert x.take_actions() == y.take_actions() and x.take_at_kyoku() == y.take_at_kyoku()
            assert x.take_at_turns() == y.take_at_turns() and x.take_shantens() == y.take_shantens()


gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(f"GPU: {gpu}", flush=True)
assert _logio.device_ready(), "the device path needs libmjx, a CUDA device and a UTF-8 locale"
_lib.init(0)
with tempfile.TemporaryDirectory() as d:
    arena = os.path.join(d, "arena")
    os.makedirs(arena)
    OneVsThree(disable_progress_bar=True, log_dir=arena).py_vs_py(Eng("challenger"), Eng("champion"), (98000, 7), args.games // 4)
    src = sorted(os.path.join(arena, f) for f in os.listdir(arena))
    print(f"arena: {len(src)} logs", flush=True)
    full = [os.path.join(d, f"full_{k:05d}.json.gz") for k in range(len(src))]
    masked = {p: [os.path.join(d, f"view{p}_{k:05d}.json.gz") for k in range(len(src))] for p in range(4)}
    pool.map(write_copies, [(fn, full[k], [masked[p][k] for p in range(4)]) for k, fn in enumerate(src)], chunksize=8)
    pool.close()
    pool.join()
    n_logs = len(src)
    print("full and masked copies written", flush=True)

    # decoder: how many masked logs it declines
    declined, decoded = 0, []
    for p in range(4):
        D = decode_dev([_logio.read_gz(f) for f in masked[p]], deltas=True)
        declined += int((~D.accept).sum())
        decoded.append(D)
    print(f"device decoder: {declined} of {4 * n_logs} masked logs declined", flush=True)

    # GameplayLoader: batches of the same files and player, masked and full alternately
    load(masked[0][:4], 0); load(full[:4], 0)  # warm-up
    stages = {"masked": [], "full": []}
    moves = 0
    for b in range(args.batches):
        p = b % 4
        lo = (b * args.batch) % max(n_logs - args.batch + 1, 1)
        got, t_m = load(masked[p][lo:lo + args.batch], p)
        want, t_f = load(full[lo:lo + args.batch], p)
        same(got, want)
        stages["masked"].append(t_m); stages["full"].append(t_f)
        moves += sum(len(gp.take_actions()) for g in got for gp in g)
        print(f"  batch {b}: seat {p}, replay + encode masked {t_m['replay + encode'] * 1e3:.1f} ms, full {t_f['replay + encode'] * 1e3:.1f} ms",
              flush=True)
    print(f"GameplayLoader(4, oracle=False, player_names=<one seat>).load_gz_log_files, {args.batches} batches of {args.batch} "
          f"files ({moves} moves), masked and full alternately, mean per batch (spread: min-max); outputs equal:")
    for key in ("read + gunzip", "decode", "replay + encode", "total"):
        m = np.array([s[key] for s in stages["masked"]]) * 1e3
        f = np.array([s[key] for s in stages["full"]]) * 1e3
        print(f"  {key:16s} masked {m.mean():8.1f} ms ({m.min():.1f}-{m.max():.1f})   full {f.mean():8.1f} ms ({f.min():.1f}-{f.max():.1f})")

# k_replay_viewpoints alone: every masked log for its own seat (4 x n_logs jobs) on the decoder's device arrays
dev = torch.device("cuda", 0)
hdr = torch.cat([D.hdr for D in decoded]); kyoku = torch.cat([D.kyoku for D in decoded])
nh = np.cumsum([0] + [D.hdr.numel() for D in decoded]); nk = np.cumsum([0] + [D.kyoku.numel() // 19 for D in decoded])
jobs = dict(hdr=hdr, kyoku=kyoku, ev_off=np.concatenate([D.ev_off + nh[p] for p, D in enumerate(decoded)]).astype(np.int32),
            ev_cnt=np.concatenate([D.ev_cnt for D in decoded]).astype(np.int32),
            ky_off=np.concatenate([D.ky_off + nk[p] for p, D in enumerate(decoded)]).astype(np.int32),
            players=np.repeat(np.arange(4, dtype=np.uint8), [len(D.ev_cnt) for D in decoded]))
env = ReplayEnv(jobs)
for _ in range(3):
    env.viewpoints()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(args.reps):
    env.viewpoints()
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / args.reps
n_ev, n_jobs = int(hdr.numel()), len(jobs["players"])
env.close()
print(f"k_replay_viewpoints ({args.reps} launches after warm-up, CUDA events): {ms:.3f} ms for {n_jobs} jobs "
      f"({n_ev} events) = {n_ev / ms / 1e3:.0f} M events/s")
