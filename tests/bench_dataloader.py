#!/usr/bin/env python
"""The trainer's input stage on arena logs (v4, file_batch_size 20, batch_size 512): (a) the reference's FileDatasetsIter restated —
this package's GameplayLoader and training_samples for populate_buffer, a host list buffer of per-move entries, random.shuffle,
torch's DataLoader collation, each batch copied to the device — against (b) mortal_b200.dataloader.FileDatasetsIter, which keeps
its buffer on the device as observation records. For each reserve_ratio the two run alternately (`--rounds` epochs each, the
order swapped every round), each epoch from the same state of `random`, and every batch of the two streams is checked equal by a
64-bit fingerprint of each tensor's bits (tests/test_gpu_dataloader.py compares them bitwise). Then k_obs_pack and k_obs_unpack
alone (CUDA events over repeated launches after warm-up) with their bytes per second against 3.35 TB/s, the bytes a buffered
sample takes and torch.cuda.max_memory_allocated. Prints the GPU name and power limit beside the numbers. Not part of the pytest
suite."""
import argparse
import os
import random
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch

import reward_lib as R
from mortal_b200.dataloader import FileDatasetsIter, pack_obs, unpack_obs
from mortal_b200.dataset import GameplayLoader
from mortal_b200.libriichi.arena import OneVsThree
from test_gpu_dataloader import PTS, RefIter

ap = argparse.ArgumentParser()
ap.add_argument("--games", type=int, default=1024, help="arena games = log files (a multiple of 4)")
ap.add_argument("--file-batch", type=int, default=20)
ap.add_argument("--batch", type=int, default=512)
ap.add_argument("--reps", type=int, default=20, help="timed codec launches")
ap.add_argument("--reserve-ratio", type=float, nargs="+", default=[0, 0.5])
ap.add_argument("--rounds", type=int, default=2, help="epochs of each path per reserve ratio; the order alternates per round")
args = ap.parse_args()
HBM = 3.35e12


class Eng:
    engine_type, version, is_oracle, enable_quick_eval, enable_rule_based_agari_guard = "mortal", 4, False, True, False

    def __init__(self, name, bias):
        self.name, self.bias = name, bias

    def react_device(self, obs, masks):
        q = torch.rand(masks.shape, device=masks.device)
        q[:, :34] += self.bias * obs[:, 876, :] + obs[:, 875, :]
        q = q.masked_fill(~masks, -1.0)
        return q.argmax(-1), q


WEIGHTS = None


def fingerprint(x):
    """a 64-bit fingerprint of a tensor's bits: their sum weighted by fixed random int64 weights (wrapping)"""
    global WEIGHTS
    v = x.reshape(-1)
    v = (v.view(torch.int32) if v.dtype == torch.float32 else v.view(torch.int64) if v.dtype == torch.float64 else v).to(torch.int64)
    if WEIGHTS is None or len(WEIGHTS) < len(v):
        g = torch.Generator(device="cpu").manual_seed(99)
        WEIGHTS = torch.randint(-2**62, 2**62, (max(len(v), 1 << 20),), generator=g, dtype=torch.int64).to(x.device)
    return (v * WEIGHTS[:len(v)]).sum()


def run_epoch(make, seed):
    """one epoch of an iterator from random.seed(seed), every batch on the device -> (per-batch fingerprints, samples, seconds to
    the last batch on the device, synchronised)"""
    random.seed(seed)
    dev = torch.device("cuda", 0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fps, n = [], 0
    for b in make():
        b = [x.to(dev, non_blocking=True) for x in b]
        n += len(b[1])
        fps.append(torch.stack([fingerprint(x) for x in b] + [torch.tensor(len(b[1]), device=dev)]))
        if len(fps) % 200 == 0:
            print(f"  {len(fps)} batches, {time.perf_counter() - t0:.1f} s", flush=True)
    torch.cuda.synchronize()
    t = time.perf_counter() - t0
    return torch.stack(fps).cpu(), n, t


gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
dev = torch.device("cuda", 0)
net = R.random_grp(64, 2, 1)
with tempfile.TemporaryDirectory() as d:
    torch.manual_seed(0)
    OneVsThree(disable_progress_bar=True, log_dir=d).py_vs_py(Eng("alpha", 2.0), Eng("beta", 0.5), (96000, 43), args.games // 4)
    files = sorted(os.path.join(d, f) for f in os.listdir(d))
    print(f"{len(files)} arena logs written", flush=True)
    results = {}
    for ratio in args.reserve_ratio:
        def ref():
            return torch.utils.data.DataLoader(RefIter(4, list(files), False, args.file_batch, ratio, 1, False, False, False, net),
                                               batch_size=args.batch, num_workers=0)

        stats = {}

        def mine():
            it = FileDatasetsIter(4, list(files), PTS, False, args.file_batch, ratio, grp=net, batch_size=args.batch)
            for b in it:
                stats["held"] = max(stats.get("held", 0), it.buffer_bytes)
                stats["record_bytes"] = it.record_bytes
                yield b

        it0 = FileDatasetsIter(4, list(files[:args.file_batch]), PTS, grp=net, batch_size=args.batch)  # warm-up of both paths
        next(iter(it0)); next(iter(ref()))
        del it0
        r = dict(ref_s=[], dev_s=[], peak_ref=0, peak_dev=0)
        for rnd in range(args.rounds):
            fp = {}
            for name in (("ref", "dev") if rnd % 2 == 0 else ("dev", "ref")):
                torch.cuda.reset_peak_memory_stats(dev)
                fp[name], n, t = run_epoch(ref if name == "ref" else mine, 7 + rnd)
                r[f"peak_{name}"] = max(r[f"peak_{name}"], torch.cuda.max_memory_allocated(dev))
                r[f"{name}_s"].append(t)
                r["n"] = n
                print(f"reserve_ratio {ratio} round {rnd} {name}: {n} samples in {t:.2f} s", flush=True)
            assert torch.equal(fp["ref"], fp["dev"]), f"streams differ (reserve_ratio {ratio}, round {rnd})"
        results[ratio] = dict(r, **stats)

    # the codec kernels alone over one file batch of loader rows
    data = GameplayLoader(4, oracle=False).load_gz_log_files(files[:args.file_batch])
    obs = torch.cat([gp.take_obs() for f in data for gp in f if len(gp._at_kyoku)])
    n = len(obs)
    rec, status = pack_obs(obs, 4)
    assert not status.any()
    idx = torch.randint(0, n, (args.batch * 8,), device=dev)
    assert torch.equal(unpack_obs(rec, torch.arange(n, device=dev), 4).view(torch.int32), obs.view(torch.int32))
    stream = torch.cuda.current_stream(dev)

    def timed(fn):
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.reps):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.reps

    out = (rec, status)
    pack_ms = timed(lambda: pack_obs(obs, 4, out=out))
    unpack_ms = timed(lambda: unpack_obs(rec, idx, 4))
    obs_b, rec_b = obs[0].numel() * 4, rec.shape[1]
    pack_bytes = n * (obs_b + rec_b + 4)
    unpack_bytes = len(idx) * (obs_b + rec_b + 8)

print(f"GPU: {gpu}")
print(f"{len(files)} v4 files, file_batch_size {args.file_batch}, batch_size {args.batch}")
for ratio, r in results.items():
    print(f"reserve_ratio {ratio}: {r['n']} samples per epoch, streams equal")
    for name, label in (("ref", "(a) reference restated (host buffer + DataLoader + copy to device)"),
                        ("dev", "(b) FileDatasetsIter (device buffer)                              ")):
        ts = r[f"{name}_s"]
        print(f"  {label}: {' / '.join(f'{t:.2f}' for t in ts)} s per epoch = {r['n'] / min(ts):,.0f} samples/s (best of {len(ts)})")
    print(f"  bytes per buffered sample {r['record_bytes']}, largest buffer {r['held'] / 2**20:.0f} MiB; "
          f"max_memory_allocated (a) {r['peak_ref'] / 2**30:.2f} GiB, (b) {r['peak_dev'] / 2**30:.2f} GiB")
print(f"k_obs_pack   {n} v4 observations: {pack_ms:.3f} ms = {pack_bytes / pack_ms / 1e9:.2f} TB/s "
      f"({pack_bytes / pack_ms / 1e9 / (HBM / 1e12):.0%} of 3.35 TB/s)")
print(f"k_obs_unpack {len(idx)} gathered observations: {unpack_ms:.3f} ms = {unpack_bytes / unpack_ms / 1e9:.2f} TB/s "
      f"({unpack_bytes / unpack_ms / 1e9 / (HBM / 1e12):.0%} of 3.35 TB/s)")
