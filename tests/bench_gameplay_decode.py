#!/usr/bin/env python
"""GameplayLoader.load_gz_log_files and Grp.load_gz_log_files: the host path (json.loads of every line, encode_events,
Grp.load_events) against the device path (thread-pool gunzip, k_mjai_decode with the deltas output, k_grp_logs, the replay from
device arrays), run alternately on the same files, with their outputs checked equal. A loader call is split into its stages:
read + gunzip, decode (host: parse + encode; device: decode + k_grp_logs + the jobs), replay + encode (the same kernels on both
paths), and Grp (host: Grp.load_events; device: the rows copied back turned into Grp objects). Also k_grp_logs alone on
device-resident arrays (CUDA events). Logs (with Mortal's per-decision `meta`) are produced on the spot by the arena, so the tool
needs no dataset. Prints the GPU name and power limit beside the numbers."""
import argparse
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from mortal_b200 import _lib, _logio
from mortal_b200.dataset import GameplayLoader, Grp
from mortal_b200.libriichi.arena import OneVsThree
from mortal_b200.validate_logs import decode_dev

ap = argparse.ArgumentParser()
ap.add_argument("--games", type=int, default=1024, help="arena games (a multiple of 4)")
ap.add_argument("--batch", type=int, default=20, help="files per load_gz_log_files call")
ap.add_argument("--batches", type=int, default=8, help="loader calls timed per path")
ap.add_argument("--reps", type=int, default=20, help="timed kernel launches")
args = ap.parse_args()


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


def _add(key, dt):
    T[key] = T.get(key, 0.0) + dt


def _wrap_load(name):
    orig = getattr(GameplayLoader, name)

    def run(self, *a):
        t0 = time.perf_counter()
        try:
            return orig(self, *a)
        finally:
            torch.cuda.synchronize()
            _add("load", time.perf_counter() - t0)

    setattr(GameplayLoader, name, run)


_orig_replay = GameplayLoader._replay


def _timed_replay(self, jobs, firsts, grps):
    def timed_grps():
        t0 = time.perf_counter()
        r = grps()
        _add("grp", time.perf_counter() - t0)
        return r

    t0 = time.perf_counter()
    r = _orig_replay(self, jobs, firsts, timed_grps)
    torch.cuda.synchronize()
    _add("replay", time.perf_counter() - t0)
    return r


_wrap_load("_load_host")
_wrap_load("_load_device")
GameplayLoader._replay = _timed_replay


def load(files, on_device):
    """one loader call -> (result, {stage: seconds})"""
    T.clear()
    ready = _logio.device_ready
    _logio.device_ready = (lambda: True) if on_device else (lambda: False)
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = GameplayLoader(4, oracle=False).load_gz_log_files(files)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
    finally:
        _logio.device_ready = ready
    return r, {"read + gunzip": total - T["load"], "decode": T["load"] - T["replay"], "replay + encode": T["replay"] - T["grp"],
               "Grp": T["grp"], "total": total}


def same(a, b):
    for pa, pb in zip(a, b, strict=True):
        for x, y in zip(pa, pb, strict=True):
            assert x.take_player_id() == y.take_player_id() and x.player_name == y.player_name
            assert torch.equal(x.take_obs(), y.take_obs()) and torch.equal(x.take_masks(), y.take_masks())
            assert x.take_actions() == y.take_actions() and x.take_at_kyoku() == y.take_at_kyoku()
            same_grp(x.take_grp(), y.take_grp())


def same_grp(a, b):
    assert np.array_equal(a.take_feature(), b.take_feature()) and a.take_rank_by_player() == b.take_rank_by_player()
    assert a.take_final_scores() == b.take_final_scores()


gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(f"GPU: {gpu}")
assert _logio.device_ready(), "the device path needs libmjx, a CUDA device and a UTF-8 locale"
_lib.init(0)
with tempfile.TemporaryDirectory() as d:
    OneVsThree(disable_progress_bar=True, log_dir=d).py_vs_py(Eng("challenger"), Eng("champion"), (98000, 7), args.games // 4)
    paths = sorted(os.path.join(d, f) for f in os.listdir(d))
    n_logs = len(paths)

    # GameplayLoader: batches of files, host and device alternately on the same files
    load(paths[:4], True); load(paths[:4], False)  # warm-up
    stages = {True: [], False: []}
    moves = 0
    for b in range(args.batches):
        files = paths[b * args.batch:(b + 1) * args.batch]
        got, t_dev = load(files, True)
        want, t_host = load(files, False)
        same(got, want)
        stages[True].append(t_dev); stages[False].append(t_host)
        moves += sum(len(gp.take_actions()) for g in got for gp in g)
    print(f"GameplayLoader(4, oracle=False).load_gz_log_files, {args.batches} batches of {args.batch} files ({moves} moves), "
          f"mean per batch; outputs equal:")
    for key in ("read + gunzip", "decode", "replay + encode", "Grp", "total"):
        h = np.mean([s[key] for s in stages[False]]) * 1e3
        dv = np.mean([s[key] for s in stages[True]]) * 1e3
        print(f"  {key:16s} host {h:9.1f} ms   device {dv:9.1f} ms")

    # Grp.load_gz_log_files on every file
    Grp.load_gz_log_files(paths[:8])
    t0 = time.perf_counter()
    got = Grp.load_gz_log_files(paths)
    t_dev = time.perf_counter() - t0
    ready = _logio.device_ready
    _logio.device_ready = lambda: False
    t0 = time.perf_counter()
    want = Grp.load_gz_log_files(paths)
    t_host = time.perf_counter() - t0
    _logio.device_ready = ready
    for a, b in zip(got, want, strict=True):
        same_grp(a, b)
    print(f"Grp.load_gz_log_files, {n_logs} files: host {t_host:.2f} s, device {t_dev:.2f} s ({t_host / t_dev:.1f}x); results equal")

    with ThreadPoolExecutor(min(32, os.cpu_count() or 1)) as pool:
        blobs = list(pool.map(_logio.read_gz, paths))

# k_grp_logs alone, device-resident arrays
L = _lib.load()
D = decode_dev(blobs, deltas=True)
assert D.accept.all(), int((~D.accept).sum())
st = torch.cuda.current_stream().cuda_stream
ptr = lambda t: t.data_ptr() if t.numel() else None
feat = torch.empty((D.kyoku.numel() // 19, 7), dtype=torch.int32, device="cuda")
rank = torch.empty((n_logs, 4), dtype=torch.uint8, device="cuda")
final = torch.empty((n_logs, 4), dtype=torch.int64, device="cuda")
status = torch.empty(n_logs, dtype=torch.int32, device="cuda")


def grp_logs():
    _lib.check(L.mjx_grp_logs_dev(n_logs, ptr(D.hdr), D.offs[0].data_ptr(), D.offs[1].data_ptr(), D.hdr.numel(), ptr(D.kyoku),
                                  D.offs[2].data_ptr(), D.kyoku.numel(), ptr(D.deltas), ptr(D.has_deltas), feat.data_ptr(),
                                  rank.data_ptr(), final.data_ptr(), status.data_ptr(), st), "grp_logs")


for _ in range(3):
    grp_logs()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(args.reps):
    grp_logs()
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / args.reps
assert not status.any()
n_ev = D.hdr.numel()
print(f"k_grp_logs ({args.reps} launches after warm-up, CUDA events): {ms:.3f} ms for {n_logs} logs = {n_ev / ms / 1e3:.0f} M events/s "
      f"({n_ev} events)")
