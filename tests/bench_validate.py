#!/usr/bin/env python
"""validate_logs throughput: the k_validate_logs kernel alone, the host decode (gunzip + JSON + word encoding), end to end, and
the oracle restatement of bin/validate_logs.rs on all host threads. Logs are produced on the spot by the arena (greedy-ish random
engine), so the tool needs no dataset. Prints the GPU name and power limit beside the numbers."""
import argparse
import concurrent.futures as cf
import gzip
import json
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

from mortal_b200 import _lib
from mortal_b200.libriichi.arena import OneVsThree
from mortal_b200.validate_logs import encode_log, pack, validate_logs

ap = argparse.ArgumentParser()
ap.add_argument("--games", type=int, default=4096, help="arena games to validate (a multiple of 4)")
ap.add_argument("--reps", type=int, default=20, help="timed kernel launches")
ap.add_argument("--cpu-logs", type=int, default=512, help="logs timed on the CPU oracle")
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
    blobs = [open(f, "rb").read() for f in files]

# host decode: gunzip + JSON + checks + word encoding
t0 = time.perf_counter()
texts = [gzip.decompress(b).decode() for b in blobs]
t1 = time.perf_counter()
enc = [encode_log(t) for t in texts]
t2 = time.perf_counter()
p = pack(enc)
t3 = time.perf_counter()
n_logs, n_ev = len(enc), int(p["ev_cnt"].sum())
print(f"{n_logs} logs, {n_ev} events ({n_ev / n_logs:.0f} per log)")
print(f"host decode: gunzip {t1 - t0:.2f} s, json + encode {t2 - t1:.2f} s, pack {t3 - t2:.3f} s = {n_logs / (t3 - t0):.0f} logs/s")

# the kernel alone: device arrays, CUDA events around repeated launches after a warm-up
L = _lib.load()
_lib.init(0)
dev = {k: torch.from_numpy(v.view(np.int64) if v.dtype == np.uint64 else v).cuda() for k, v in p.items()}
out = torch.zeros((n_logs, 4), dtype=torch.int32, device="cuda")
st = torch.cuda.current_stream()


def launch():
    _lib.check(L.mjx_validate_logs_dev(n_logs, dev["hdr"].data_ptr(), dev["ev_off"].data_ptr(), dev["ev_cnt"].data_ptr(), len(p["hdr"]),
                                       dev["kyoku"].data_ptr(), dev["ky_off"].data_ptr(), len(p["kyoku"]), dev["hora"].data_ptr(),
                                       dev["hora_off"].data_ptr(), len(p["hora"]), out.data_ptr(), st.cuda_stream), "validate")


for _ in range(3):
    launch()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(args.reps):
    launch()
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / args.reps
assert (out[:, 0] == 0).all(), "arena logs must be valid"
print(f"kernel: {ms:.2f} ms per launch = {n_logs / ms * 1e3:.0f} logs/s, {n_ev / ms * 1e3 / 1e6:.1f} M events/s")

# end to end: gz bytes in memory -> verdicts
torch.cuda.synchronize()
t0 = time.perf_counter()
v = validate_logs([gzip.decompress(b).decode() for b in blobs])
dt = time.perf_counter() - t0
assert v == [None] * n_logs
print(f"end to end: {dt:.2f} s = {n_logs / dt:.0f} logs/s")

# the oracle restatement on all host threads (the ctypes call releases the GIL); JSON decoding outside the timed window
import oracle_lib as O
import validate_lib as VL

sub = []
for t in texts[: args.cpu_logs]:
    evs = [json.loads(x) for x in t.splitlines() if x.strip()]
    sub.append((VL.oracle_events(evs), len(evs)))
O.lib()
cores = len(os.sched_getaffinity(0))
t0 = time.perf_counter()
with cf.ThreadPoolExecutor(cores) as ex:
    res = list(ex.map(lambda job: VL.oracle_validate_events(*job), sub))
dt = time.perf_counter() - t0
assert all(r[0] == 0 for r in res)
print(f"oracle: {len(sub)} logs in {dt:.2f} s = {len(sub) / dt:.0f} logs/s on {cores} host threads (decoded events in, verdicts out)")
