#!/usr/bin/env python
"""mjai decode throughput: the k_mjai_decode count + fill kernels alone (device-resident text), the host decoder (json.loads +
checks + word encoding) against the device decoder from text in host memory, and end-to-end validate_logs with the gunzip and
file-read stages beside it. Logs (with Mortal's per-decision `meta`) are produced on the spot by the arena, so the tool needs no
dataset. Prints the GPU name and power limit beside the numbers."""
import argparse
import gzip
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

from mortal_b200 import _lib
from mortal_b200.libriichi.arena import OneVsThree
from mortal_b200.validate_logs import decode_dev, encode_log, validate_logs

ap = argparse.ArgumentParser()
ap.add_argument("--games", type=int, default=1024, help="arena games (a multiple of 4)")
ap.add_argument("--reps", type=int, default=20, help="timed kernel launches")
args = ap.parse_args()


class Eng:
    engine_type, version, is_oracle, enable_quick_eval, enable_rule_based_agari_guard, name = "mortal", 4, False, True, False, "e"

    def react_device(self, obs, masks):
        q = torch.rand(masks.shape, device=masks.device)
        q[:, :34] += 2.0 * obs[:, 876, :] + obs[:, 875, :]
        q = q.masked_fill(~masks, -1.0)
        return q.argmax(-1), q


gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(f"GPU: {gpu}")
with tempfile.TemporaryDirectory() as d:
    OneVsThree(disable_progress_bar=True, log_dir=d).py_vs_py(Eng(), Eng(), (91000, 7), args.games // 4)
    files = sorted(os.path.join(d, f) for f in os.listdir(d))
    t0 = time.perf_counter()
    with ThreadPoolExecutor(min(32, os.cpu_count() or 1)) as pool:
        blobs_gz = list(pool.map(lambda f: open(f, "rb").read(), files))
    t_read = time.perf_counter() - t0

t0 = time.perf_counter()
texts = [gzip.decompress(b).decode() for b in blobs_gz]
t_gunzip = time.perf_counter() - t0
with ThreadPoolExecutor(min(32, os.cpu_count() or 1)) as pool:
    t0 = time.perf_counter()
    list(pool.map(lambda b: gzip.decompress(b).decode(), blobs_gz))
    t_gunzip_pool = time.perf_counter() - t0
blobs = [t.encode() for t in texts]
n_logs, n_bytes = len(blobs), sum(len(b) for b in blobs)
print(f"{n_logs} logs, {n_bytes / 1e6:.1f} MB of text; file reads {t_read:.3f} s; gunzip {t_gunzip:.2f} s serial, "
      f"{t_gunzip_pool:.2f} s on a thread pool")

# host decoder
t0 = time.perf_counter()
enc = [encode_log(t) for t in texts]
t_host = time.perf_counter() - t0
n_ev = sum(len(e.hdr) for e in enc)
print(f"host decode (json.loads + checks + words): {t_host:.2f} s = {n_logs / t_host:.0f} logs/s ({n_ev} events)")

# device decoder from host text (H2D, count, the counts' D2H, fill)
_lib.init(0)
decode_dev(blobs[:8])
torch.cuda.synchronize()
t0 = time.perf_counter()
D = decode_dev(blobs)
torch.cuda.synchronize()
t_dev = time.perf_counter() - t0
declined = int((~D.accept).sum())
print(f"device decode from host text: {t_dev * 1e3:.1f} ms = {n_logs / t_dev:.0f} logs/s; declined logs: {declined}")
assert int(D.ev_cnt.sum()) == n_ev

# the kernels alone: device-resident text, CUDA events around repeated count + fill launches
L = _lib.load()
dev = torch.device("cuda", 0)
st = torch.cuda.current_stream().cuda_stream
log_off = np.zeros(n_logs + 1, dtype=np.int64)
np.cumsum([len(b) for b in blobs], out=log_off[1:])
text = torch.frombuffer(bytearray(b"".join(blobs)), dtype=torch.uint8).to(dev)
d_off = torch.from_numpy(log_off).to(dev)
counts = torch.empty((n_logs, 6), dtype=torch.int32, device=dev)


def count():
    _lib.check(L.mjx_mjai_count_dev(n_logs, text.data_ptr(), n_bytes, d_off.data_ptr(), 0, counts.data_ptr(), st), "count")


def fill():
    _lib.check(L.mjx_mjai_fill_dev(n_logs, text.data_ptr(), n_bytes, d_off.data_ptr(), 0, counts.data_ptr(), D.offs[0].data_ptr(),
                                   D.offs[2].data_ptr(), D.offs[3].data_ptr(), D.hdr.data_ptr(), D.lines.data_ptr(), D.hdr.numel(),
                                   D.kyoku.data_ptr(), D.kyoku.numel(), D.hora.data_ptr(), D.hora.numel(), st), "fill")


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


ms_count, ms_fill = timed(count), timed(fill)
ms = ms_count + ms_fill
print(f"kernels: count {ms_count:.2f} ms + fill {ms_fill:.2f} ms = {ms:.2f} ms = {n_logs / ms * 1e3:.0f} logs/s, "
      f"{n_bytes / ms / 1e6:.1f} GB/s of text")

# end to end: gz bytes in memory -> verdicts, and the same from decompressed text
torch.cuda.synchronize()
t0 = time.perf_counter()
with ThreadPoolExecutor(min(32, os.cpu_count() or 1)) as pool:
    v = validate_logs(list(pool.map(lambda b: gzip.decompress(b).decode(), blobs_gz)))
dt = time.perf_counter() - t0
assert v == [None] * n_logs
t0 = time.perf_counter()
validate_logs(texts)
dt_text = time.perf_counter() - t0
print(f"validate_logs end to end: {dt:.2f} s = {n_logs / dt:.0f} logs/s from gz bytes (thread-pool gunzip); "
      f"{dt_text:.2f} s = {n_logs / dt_text:.0f} logs/s from decompressed text")
