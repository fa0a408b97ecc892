#!/usr/bin/env python
"""Forward time per step of Mortal networks of every version (and the version-4 oracle brain) at 192 x 40 on ~4,096 arena rows:
the fused device path (Brain.prepare_fast / forward_fast, csrc/mjx_nn.cuh) against the stock module under bf16 autocast, which is
what DeviceEngine runs for a module without prepare_fast; and OneVsThree.py_vs_py table-steps/s for a version-1 engine against a
version-4 one. Prints the card and its power limit with the numbers, one JSON line at the end.

usage: python tests/bench_checkpoint_engine.py [--rows 4096] [--iters 20] [--seeds 256]"""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def card():
    import torch

    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except OSError:
        q = ""
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def arena_rows(n_rows):
    import torch

    import mortal_b200

    n = n_rows
    env = mortal_b200.BatchEnv(np.repeat(np.arange(60000, 60000 + n // 4, dtype=np.uint64), 4), np.full(n, 0x2000, dtype=np.uint64))
    actions = torch.zeros(env.row_cap, dtype=torch.int64, device=env.device)
    rows, want = {v: [] for v in (1, 2, 3, 4)}, n_rows
    inv4, masks = [], []
    env.step(None)
    got = 0
    while got < want:
        nr = env.num_rows()
        for v in (1, 2, 3, 4):
            env.set_obs_version(v)
            rows[v].append(env.encode_obs()[:nr].clone())
        inv4.append(env.encode_invisible(4)[:nr].clone())
        masks.append(env.masks[:nr].clone().bool())
        got += nr
        env.set_obs_version(4)
        env.policy_test(1, actions)
        env.step(actions)
    env.close()
    cat = lambda xs: torch.cat(xs)[:want].contiguous()
    return {v: cat(x) for v, x in rows.items()}, cat(inv4), cat(masks)


def time_ms(fn, iters):
    import torch

    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--seeds", type=int, default=256)
    args = ap.parse_args()
    import torch

    import mortal_b200
    import mortal_b200.libriichi as lr
    from mortal_b200.engine import DeviceEngine
    from mortal_b200.model import DQN, Brain

    mortal_b200._lib.init(0)
    dev = torch.device("cuda", 0)
    info = card()
    print("card:", info, flush=True)
    rows, inv, masks = arena_rows(args.rows)
    out = {"card": info, "rows": int(masks.shape[0]), "forward_ms": {}}
    for name, version, oracle in (("v1", 1, False), ("v2", 2, False), ("v3", 3, False), ("v4", 4, False), ("v4_oracle", 4, True)):
        torch.manual_seed(version)
        brain = Brain(conv_channels=192, num_blocks=40, version=version, is_oracle=oracle).to(dev).eval()
        obs = rows[version]
        extra = (inv,) if oracle else ()
        fast = copy.deepcopy(brain)
        with torch.no_grad():
            fast.prepare_fast(torch.bfloat16)

        def run_fast():
            with torch.inference_mode():
                fast.forward_fast(obs, *extra)

        def run_stock():
            with torch.inference_mode(), torch.autocast("cuda", dtype=torch.bfloat16):
                brain(obs, *extra)

        f, s = time_ms(run_fast, args.iters), time_ms(run_stock, args.iters)
        out["forward_ms"][name] = {"fused": round(f, 3), "stock_autocast": round(s, 3), "speedup": round(s / f, 2)}
        print(name, out["forward_ms"][name], flush=True)
        del brain, fast
        torch.cuda.empty_cache()
    lr.install()
    from libriichi.arena import OneVsThree

    torch.manual_seed(0)
    mk = lambda v: DeviceEngine(Brain(conv_channels=192, num_blocks=40, version=v), DQN(version=v), version=v, device=dev, name=f"v{v}")
    a, b = mk(1), mk(4)
    arena = OneVsThree(disable_progress_bar=True, log_dir=None)
    arena.py_vs_py(challenger=a, champion=b, seed_start=(70000, 0x2000), seed_count=8)  # warm-up
    torch.cuda.synchronize()
    t = time.perf_counter()
    arena.py_vs_py(challenger=a, champion=b, seed_start=(71000, 0x2000), seed_count=args.seeds)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t
    steps = arena.last_stats["table_steps"]
    out["py_vs_py_v1_vs_v4"] = {"games": 4 * args.seeds, "table_steps": steps, "seconds": round(dt, 2), "table_steps_per_s": round(steps / dt)}
    print("py_vs_py v1 vs v4:", out["py_vs_py_v1_vs_v4"], flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
