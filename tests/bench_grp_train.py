#!/usr/bin/env python
"""GRP training throughput: the reference's train_grp.py step against the device path (not part of the pytest suite).

    python tests/bench_grp_train.py [--games 256] [--steps 100] [--warmup 10] [--out DIR]

Generates arena logs on the spot (`--games` sets of 4 hanchan: 1,024 logs by default), then times two arms, each over `--steps`
training steps after `--warmup`, every window ending in a device synchronise:
  (a) the reference as train_grp.py runs it: the restated GrpFileDatasetsIter in a DataLoader(num_workers=1, collate_fn=collate)
      (pad_sequence + pack_padded_sequence per batch), torch's float64 GRU on the GPU, cross_entropy, backward, AdamW; its logs
      are decoded once up front, so its loader is timed without log decoding (the device arm's loading is timed);
  (b) GrpFileDatasetsIter + grp_loss + the same AdamW, decoding every file batch's logs as it loads them (Grp.load_gz_log_files);
  (c) (b) over the reference arm's pre-decoded logs, the equal-footing comparison with (a).
Both use batch 512, file_batch_size 50 and the default GRP (hidden 64, 2 layers). It also reports the device kernels' time per
step from CUDA events around grp_loss, and checks that both arms reach the same weights over the same sample stream (driven with
num_workers=0 for that check). The GPU name and power limit are printed beside the numbers."""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
from torch.nn import functional as F
from torch.nn.utils.rnn import pack_padded_sequence, pad_sequence
from torch.utils.data import DataLoader, IterableDataset

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import grp_train_lib as T  # noqa: E402
from mortal_b200.dataset import Grp  # noqa: E402
from mortal_b200 import grp_train  # noqa: E402
from mortal_b200.grp_train import GrpFileDatasetsIter, grp_loss  # noqa: E402
from mortal_b200.model import GRP  # noqa: E402
from test_gpu_gameplay_decode import _Eng  # noqa: E402


class RefDataset(IterableDataset):
    """the restated GrpFileDatasetsIter over `cache` (file -> (feature, rank_by_player)), decoded once before the loaders start,
    so the reference arm's loading costs nothing; picklable for a spawned worker (a forked one cannot use CUDA for pinning)"""

    def __init__(self, files, cache, cycle=True):
        self.files, self.cache, self.cycle = files, cache, cycle

    def load(self, chunk):
        return [self.cache[f] for f in chunk]

    def __iter__(self):
        return iter(T.RefGrpFileDatasetsIter(self.files, self.load, 50, self.cycle))


def collate(batch):  # train_grp.py collate
    inputs, lengths, ranks = [], [], []
    for seq, rank in batch:
        inputs.append(seq)
        lengths.append(len(seq))
        ranks.append(rank)
    lengths = torch.tensor(lengths)
    ranks = torch.tensor(ranks, dtype=torch.int64, pin_memory=True)
    packed = pack_padded_sequence(pad_sequence(inputs, batch_first=True), lengths, batch_first=True, enforce_sorted=False)
    packed.pin_memory()
    return packed, ranks


def ref_step(grp, opt, packed, ranks):
    packed = packed.to(dtype=torch.float64, device="cuda")
    ranks = ranks.to(dtype=torch.int64, device="cuda")
    _, state = grp.rnn(packed)
    logits = grp.fc(state.transpose(0, 1).flatten(1))
    mappings = (grp.perms.expand(len(ranks), -1, -1).transpose(0, 1) == ranks).all(-1).nonzero()
    labels = torch.zeros(len(ranks), dtype=torch.int64, device="cuda")
    labels[mappings[:, 1]] = mappings[:, 0]
    loss = F.cross_entropy(logits, labels)
    opt.zero_grad(set_to_none=True)
    loss.backward()
    opt.step()
    return loss


def time_arm(step, batches, steps, warmup):
    for _ in range(warmup):
        step(next(batches))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        step(next(batches))
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, default=256)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--check-steps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from mortal_b200.libriichi.arena import OneVsThree

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    d = tempfile.mkdtemp(prefix="bench_grp_train_")
    OneVsThree(disable_progress_bar=True, log_dir=d).py_vs_py(_Eng("alpha", 2.0), _Eng("beta", 0.5), (96000, 43), a.games)
    files = sorted(os.path.join(d, f) for f in os.listdir(d))
    grps = dict(zip(files, Grp.load_gz_log_files(files)))
    cache = {f: (g.take_feature(), g.take_rank_by_player()) for f, g in grps.items()}
    n_rows = sum(len(v[0]) for v in cache.values())
    print(f"{len(files)} logs, {n_rows} kyoku rows (= samples per epoch); GPU: {gpu}", flush=True)

    torch.manual_seed(0)
    init = GRP()
    # (a) the reference arm
    random.seed(1)
    ref = T.RefGRP().cuda()
    ref.load_state_dict(init.state_dict())
    opt_r = torch.optim.AdamW(ref.parameters())
    loader = iter(DataLoader(RefDataset(list(files), cache), batch_size=512, drop_last=True, num_workers=1, collate_fn=collate,
                             multiprocessing_context="spawn"))
    t_ref = time_arm(lambda b: ref_step(ref, opt_r, *b), loader, a.steps, a.warmup)
    del loader
    # (b) the device arm, with CUDA events around the kernels in a second window
    random.seed(1)
    dev = GRP().cuda()
    dev.load_state_dict(init.state_dict())
    opt_d = torch.optim.AdamW(dev.parameters())

    def dev_step(b):
        opt_d.zero_grad(set_to_none=True)
        grp_loss(dev, b)
        opt_d.step()

    it = iter(GrpFileDatasetsIter(list(files), 50, True, batch_size=512))
    t_dev = time_arm(dev_step, it, a.steps, a.warmup)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.steps)]
    for e0, e1 in ev:
        b = next(it)
        opt_d.zero_grad(set_to_none=True)
        e0.record()
        grp_loss(dev, b)
        e1.record()
        opt_d.step()
    torch.cuda.synchronize()
    kern_ms = float(np.mean([e0.elapsed_time(e1) for e0, e1 in ev]))
    # (c) the device arm over the same pre-decoded logs as the reference arm: the iterator, grp_loss and AdamW alone
    class Decoded:
        load_gz_log_files = staticmethod(lambda chunk: [grps[f] for f in chunk])

    grp_train.Grp = Decoded
    it = iter(GrpFileDatasetsIter(list(files), 50, True, batch_size=512))
    t_dev_decoded = time_arm(dev_step, it, a.steps, a.warmup)
    grp_train.Grp = Grp

    # agreement over one sample stream (num_workers=0, so both arms draw the same batches)
    random.seed(7)
    ref_stream = list(zip(range(a.check_steps), DataLoader(RefDataset(list(files), cache), batch_size=512, drop_last=True, num_workers=0,
                                                           collate_fn=collate)))
    random.seed(7)
    it = iter(GrpFileDatasetsIter(list(files), 50, True, batch_size=512))
    dev_stream = [next(it) for _ in range(a.check_steps)]
    ref.load_state_dict(init.state_dict())
    dev.load_state_dict(init.state_dict())
    opt_r = torch.optim.AdamW(ref.parameters(), lr=1e-3)
    opt_d = torch.optim.AdamW(dev.parameters(), lr=1e-3)
    for (_, b), db in zip(ref_stream, dev_stream):
        ref_step(ref, opt_r, *b)
        opt_d.zero_grad(set_to_none=True)
        grp_loss(dev, db)
        opt_d.step()
    gap = max((p - q).abs().max().item() for p, q in zip(dev.parameters(), ref.parameters()))

    res = dict(gpu=gpu, logs=len(files), batch=512, steps=a.steps, ref_steps_per_s=a.steps / t_ref, dev_steps_per_s=a.steps / t_dev,
               dev_predecoded_steps_per_s=a.steps / t_dev_decoded, speedup_predecoded=t_ref / t_dev_decoded, dev_kernel_ms_per_step=kern_ms, check_steps=a.check_steps, max_param_gap=gap)
    print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_grp_train.json"), "w") as f:
            json.dump(res, f, indent=1)
    assert gap <= 1e-9, gap


if __name__ == "__main__":
    main()
