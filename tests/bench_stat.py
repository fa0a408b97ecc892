#!/usr/bin/env python
"""Stat.from_dir throughput: the host path (json.loads of every line + Stat.from_game per seat) against the device path
(thread-pool gunzip, k_mjai_decode with the deltas output, k_stat_logs) end to end on the same directory, the file reads + gunzip
stage alone, and the kernels alone on device-resident arrays (CUDA events): the deltas fill against the plain fill, and
k_stat_logs. Logs (with Mortal's per-decision `meta`) are produced on the spot by the arena with two engine names, so the tool
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

from mortal_b200 import _lib, stat
from mortal_b200.libriichi.arena import OneVsThree
from mortal_b200.validate_logs import decode_dev

ap = argparse.ArgumentParser()
ap.add_argument("--games", type=int, default=1024, help="arena games (a multiple of 4)")
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


gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(f"GPU: {gpu}")
assert stat._device_ready(), "the device path needs libmjx and a CUDA device"
_lib.init(0)
with tempfile.TemporaryDirectory() as d:
    OneVsThree(disable_progress_bar=True, log_dir=d).py_vs_py(Eng("challenger"), Eng("champion"), (97000, 5), args.games // 4)
    paths = stat._log_paths(d)
    n_logs = len(paths)

    # file reads + gunzip on the thread pool (what the device path does first)
    t0 = time.perf_counter()
    with ThreadPoolExecutor(min(32, os.cpu_count() or 1)) as pool:
        blobs = list(pool.map(stat._read_bytes, paths))
    t_read = time.perf_counter() - t0
    n_bytes = sum(len(b) for b in blobs)
    print(f"{n_logs} logs, {n_bytes / 1e6:.1f} MB of text; file reads + gunzip on a thread pool: {t_read:.2f} s")

    # end to end: host path, then device path (warmed up on a few files first)
    t0 = time.perf_counter()
    host = stat.Stat()
    for p in paths:
        host = host + stat._host_log_stat(p, "challenger")
    t_host = time.perf_counter() - t0
    stat._device_from_dir(paths[:8], "challenger")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    dev = stat.Stat.from_dir(d, "challenger")
    t_dev = time.perf_counter() - t0
    assert repr(dev) == repr(host), (dev, host)
    print(f"Stat.from_dir end to end: host {t_host:.2f} s = {n_logs / t_host:.0f} logs/s; device {t_dev:.2f} s = "
          f"{n_logs / t_dev:.0f} logs/s; {t_host / t_dev:.1f}x; results equal")

# the kernels alone, device-resident arrays
L = _lib.load()
D = decode_dev(blobs, deltas=True)
assert D.accept.all(), int((~D.accept).sum())
st = torch.cuda.current_stream().cuda_stream
log_off = np.zeros(n_logs + 1, dtype=np.int64)
np.cumsum([len(b) for b in blobs], out=log_off[1:])
text = torch.frombuffer(bytearray(b"".join(blobs)), dtype=torch.uint8).cuda()
d_off = torch.from_numpy(log_off).cuda()
counts = torch.from_numpy(D.counts).cuda()
ptr = lambda t: t.data_ptr() if t.numel() else None
seats = torch.full((n_logs,), 15, dtype=torch.uint8, device="cuda")
out = torch.empty((n_logs, len(stat.COUNTERS)), dtype=torch.int64, device="cuda")
status = torch.empty(n_logs, dtype=torch.int32, device="cuda")


def fill():
    _lib.check(L.mjx_mjai_fill_dev(n_logs, text.data_ptr(), n_bytes, d_off.data_ptr(), 0, counts.data_ptr(), D.offs[0].data_ptr(),
                                   D.offs[2].data_ptr(), D.offs[3].data_ptr(), ptr(D.hdr), ptr(D.lines), D.hdr.numel(),
                                   ptr(D.kyoku), D.kyoku.numel(), ptr(D.hora), D.hora.numel(), st), "fill")


def fill_deltas():
    _lib.check(L.mjx_mjai_fill_deltas_dev(n_logs, text.data_ptr(), n_bytes, d_off.data_ptr(), 0, counts.data_ptr(),
                                          D.offs[0].data_ptr(), D.offs[2].data_ptr(), D.offs[3].data_ptr(), ptr(D.hdr), ptr(D.lines),
                                          D.hdr.numel(), ptr(D.kyoku), D.kyoku.numel(), ptr(D.hora), D.hora.numel(), ptr(D.deltas),
                                          ptr(D.has_deltas), st), "fill_deltas")


def stat_logs():
    _lib.check(L.mjx_stat_logs_dev(n_logs, ptr(D.hdr), D.offs[0].data_ptr(), D.offs[1].data_ptr(), D.hdr.numel(), ptr(D.kyoku),
                                   D.offs[2].data_ptr(), D.kyoku.numel(), ptr(D.deltas), ptr(D.has_deltas), seats.data_ptr(),
                                   out.data_ptr(), status.data_ptr(), st), "stat_logs")


def timed(fn):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / args.reps


ms = {}
for _ in range(2):  # alternate the two fills so drift affects both alike
    for name, fn in (("fill", fill), ("fill_deltas", fill_deltas)):
        ms.setdefault(name, []).append(timed(fn))
ms_stat = timed(stat_logs)
assert not status.any()
n_ev = D.hdr.numel()
print(f"kernels ({args.reps} launches after warm-up, CUDA events): plain fill {min(ms['fill']):.2f} ms, deltas fill "
      f"{min(ms['fill_deltas']):.2f} ms (runs: {', '.join(f'{x:.2f}' for x in ms['fill'])} / "
      f"{', '.join(f'{x:.2f}' for x in ms['fill_deltas'])}); k_stat_logs (all four seats) {ms_stat:.3f} ms = "
      f"{n_ev / ms_stat / 1e3:.0f} M events/s ({n_ev} events)")
