#!/usr/bin/env python
"""OneVsThree.py_vs_py with log_dir: the host writer (mjai_log.write_logs) against the device writer (mortal_b200/mjai_write.py) on
the same seeds, beside the run without logs, with a deterministic device engine (Q a function of the observation). Checks that both
writers produce the same files, prints the device writer's stages and the render kernels' times (CUDA events over repeated launches),
and the GPU name and power limit beside the numbers.

    python tests/bench_arena_logs.py --games 1024 [--device-only]
"""
import argparse
import ctypes as C
import gzip
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, default=1024)
    ap.add_argument("--device-only", action="store_true", help="skip the host writer leg")
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    import torch

    import mortal_b200
    from mortal_b200 import _lib
    from mortal_b200.libriichi.arena import OneVsThree
    from test_gpu_arena_logs import DevEngine

    _lib.init(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(f"GPU: {gpu}; {os.cpu_count()} host CPUs")
    seeds = a.games // 4
    chal, champ = DevEngine(torch, "a", salt=0.1), DevEngine(torch, "b")
    tmp = tempfile.mkdtemp()
    out = {}

    import types

    from mortal_b200.libriichi import arena as A

    def run(tag, log_dir, host=False, meta=True):
        clock = iter(range(10 ** 6, 10 ** 15, 1237))  # a counter for eval_time_ns, so both writers' outputs can be compared
        A.time = types.SimpleNamespace(perf_counter_ns=lambda: next(clock))
        ar = OneVsThree(disable_progress_bar=True, log_dir=log_dir)
        ar.host_log_writer = host
        ar.log_meta = meta
        torch.manual_seed(0)
        torch.cuda.synchronize()
        t = time.perf_counter()
        ar.py_vs_py(chal, champ, (20000, 7), seeds)
        torch.cuda.synchronize()
        out[tag] = time.perf_counter() - t
        print(f"{tag}: {out[tag]:.2f} s ({ar.last_stats['cycles']} cycles)", flush=True)
        return ar

    run("warmup", None)
    run("no_logs", None)
    plain = run("device_logs_without_meta", os.path.join(tmp, "plain"), meta=False)
    dev = run("device_logs", os.path.join(tmp, "dev"))
    cycles = dev.last_stats["cycles"]
    n_rec = dev.last_meta_records
    print("device writer stages (s):", {k: round(v, 3) for k, v in dev.last_log_timing.items()})
    print(f"records: {n_rec} decision rows, {n_rec * 221 / 2 ** 20:.0f} MiB on the device while playing (221 B each); "
          f"recording + meta rendering over the meta-free device run: "
          f"{(out['device_logs'] - out['device_logs_without_meta']) / cycles * 1e3:.3f} ms per cycle")
    text_bytes = sum(len(gzip.open(p).read()) for p in dev.last_log_paths[:64]) * len(dev.last_log_paths) / 64
    if not a.device_only:
        host = run("host_logs", os.path.join(tmp, "host"), host=True)
        same = all(gzip.open(x).read() == gzip.open(y).read() for x, y in zip(dev.last_log_paths, host.last_log_paths))
        print(f"outputs equal: {same} over {len(dev.last_log_paths)} files")
        assert same
    print(f"logging overhead: device {out['device_logs'] - out['no_logs']:.2f} s"
          + ("" if a.device_only else f", host {out['host_logs'] - out['no_logs']:.2f} s")
          + f"; ~{text_bytes / 2 ** 20:.0f} MiB of text")
    # the render kernels alone over a finished batch's log (no meta), CUDA events over repeated launches
    n = a.games
    env = mortal_b200.BatchEnv(np.repeat(np.arange(20000, 20000 + seeds, dtype=np.uint64), 4), np.full(n, 7, dtype=np.uint64))
    env.enable_log()
    env.run_test_policy(1)
    L = _lib.load()
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    common = (n, C.c_void_p(env.log_words.data_ptr()), C.c_void_p(env.log_len.data_ptr()), env._log_cap, None, 0, 1, None, None, None,
              None, None, 0)
    nb = torch.empty(n, dtype=torch.int32, device="cuda")
    st = torch.empty(n, dtype=torch.int32, device="cuda")

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / a.reps

    # k_meta_record over every row a step emits, random Q-values, v4 observation (shanten / furiten)
    env2 = mortal_b200.BatchEnv(np.repeat(np.arange(20000, 20000 + seeds, dtype=np.uint64), 4), np.full(n, 7, dtype=np.uint64))
    env2.enable_log()
    env2.step(None)
    nr = env2.num_rows()
    obs = env2.encode_obs()
    from mortal_b200.mjai_write import DeviceMetaRecorder

    rec = DeviceMetaRecorder(n, 4, env2)
    rec._alloc(max(rec.cap, nr * (a.reps + 1)))
    qr = torch.randn((nr, 46), device="cuda")
    acts = torch.zeros(env2.row_cap, dtype=torch.int64, device="cuda")
    ms_rec = timed(lambda: rec.record(0, nr, qr, acts, call=0, obs=obs))
    assert rec.error is None and rec.count == nr * (a.reps + 1)
    env2.close()
    ms_count = timed(lambda: _lib.check(L.mjx_mjai_render_count_dev(*common, C.c_void_p(nb.data_ptr()), C.c_void_p(st.data_ptr()), sp)))
    nb_h = nb.cpu().numpy().astype(np.int64)
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(nb_h)])).cuda()
    buf = torch.empty(int(nb_h.sum()), dtype=torch.uint8, device="cuda")
    ms_fill = timed(lambda: _lib.check(L.mjx_mjai_render_fill_dev(*common, C.c_void_p(st.data_ptr()), C.c_void_p(off.data_ptr()), 0, n,
                                                                   C.c_void_p(buf.data_ptr()), buf.numel(), sp)))
    pinned = torch.empty(buf.numel(), dtype=torch.uint8, pin_memory=True)
    ms_d2h = timed(lambda: pinned.copy_(buf, non_blocking=True))
    env.close()
    print(f"k_meta_record over {nr} rows: {ms_rec:.4f} ms")
    print(f"render kernels, {n} games without meta, {buf.numel() / 2 ** 20:.0f} MiB: count {ms_count:.2f} ms, fill {ms_fill:.2f} ms, "
          f"D2H {ms_d2h:.2f} ms")
    print(json.dumps(dict(gpu=gpu, games=a.games, **{k: round(v, 3) for k, v in out.items()},
                          stages={k: round(v, 3) for k, v in dev.last_log_timing.items()}, count_ms=round(ms_count, 3), meta_record_ms=round(ms_rec, 4), meta_record_rows=nr, records=n_rec,
                          fill_ms=round(ms_fill, 3), d2h_ms=round(ms_d2h, 3))))
    shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
