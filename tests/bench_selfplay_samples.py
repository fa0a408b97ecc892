#!/usr/bin/env python
"""Training samples from self-play: the log round trip against the device words (not part of the pytest suite).

    python tests/bench_selfplay_samples.py [--games 800] [--rounds 3] [--batch-size 512] [--file-batch-size 20]

Plays one OneVsThree session of `--games` games (rounded down to whole seeds) with `record_games` and `log_dir` both on, so the
written files and `last_games` come from the same run, then runs two arms alternately, `--rounds` times each:
  (a) FileDatasetsIter over the written files (read, gunzip, device decode, replay), as online training over a drained directory;
  (b) SelfPlayDatasetsIter over `last_games` (k_arena_words, replay), which writes and reads no file.
Each arm iterates to its last batch (trainee samples, the reference profile's dataset flags) and ends in a device synchronise.
Before timing, both streams are compared batch by batch for the same random state. It prints, as one JSON line, each arm's
median seconds per pass and samples/s, the converter's kernel time per pass over all games (CUDA events around
mjx_arena_words_count_dev + mjx_arena_words_fill_dev), and the GPU's name and power limit read in the same run. The session's
play time is not part of either arm: both need the games."""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import reward_lib as R  # noqa: E402
from mortal_b200 import _lib  # noqa: E402
from mortal_b200.dataloader import FileDatasetsIter  # noqa: E402
from mortal_b200.libriichi.arena import OneVsThree  # noqa: E402
from mortal_b200.selfplay import SelfPlayDatasetsIter, _load, decode_games  # noqa: E402
from test_gpu_gameplay_decode import _Eng  # noqa: E402

PTS = [6.0, 4.0, 2.0, 0.0]


def _iters(games, paths, grp, args):
    kw = dict(file_batch_size=args.file_batch_size, reserve_ratio=0.0, player_names=["trainee"], grp=grp, batch_size=args.batch_size)
    return (lambda: FileDatasetsIter(4, list(paths), PTS, **kw)), (lambda: SelfPlayDatasetsIter(4, games, PTS, **kw))


def check_equal(make_a, make_b, seed):
    """both streams in lockstep, each with its own copy of `random`'s state -> the number of batches (AssertionError on a difference)"""
    random.seed(seed)
    st = [random.getstate()] * 2
    its = [iter(make_a()), iter(make_b())]
    n = 0
    while True:
        out = []
        for k in range(2):
            random.setstate(st[k])
            out.append(next(its[k], None))
            st[k] = random.getstate()
        if out[0] is None or out[1] is None:
            assert out[0] is None and out[1] is None, "the streams differ in length"
            return n
        for x, y in zip(*out):
            assert x.dtype == y.dtype and torch.equal(x, y), f"batch {n} differs"
        n += 1


def run_arm(make, seed):
    random.seed(seed)
    torch.cuda.synchronize()
    t = time.perf_counter()
    n = 0
    for b in make():
        n += b[0].shape[0]
    torch.cuda.synchronize()
    return time.perf_counter() - t, n


def converter_ms(games, reps=20):
    """mean device time of one count + fill launch pair over all games (the buffers sized once by decode_games)"""
    L = _load()
    D = decode_games(games)
    dev = games.words.device
    st = torch.cuda.current_stream(dev).cuda_stream
    words, lens = games.words.contiguous(), games.lens.to(torch.int32).contiguous()
    counts = torch.empty((len(games), 4), dtype=torch.int32, device=dev)
    n = len(games)

    def launch():
        _lib.check(L.mjx_arena_words_count_dev(n, words.data_ptr(), lens.data_ptr(), words.shape[1], games.log_cap, counts.data_ptr(), st))
        _lib.check(L.mjx_arena_words_fill_dev(n, words.data_ptr(), lens.data_ptr(), words.shape[1], games.log_cap, 0, counts.data_ptr(),
                                              D.offs[0].data_ptr(), D.offs[2].data_ptr(), D.offs[3].data_ptr(), D.hdr.data_ptr(),
                                              D.lines.data_ptr(), D.hdr.numel(), D.kyoku.data_ptr(), D.kyoku.numel(), D.hora.data_ptr(),
                                              D.hora.numel(), D.deltas.data_ptr(), D.has_deltas.data_ptr(), st))

    launch()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        launch()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, default=800)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch-size", type=int, default=512)
    ap.add_argument("--file-batch-size", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_selfplay_samples needs a CUDA device")
    _lib.init(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    grp = R.random_grp(64, 2, 21)
    with tempfile.TemporaryDirectory() as d:
        arena = OneVsThree(disable_progress_bar=True, log_dir=d)
        arena.record_games = True
        torch.manual_seed(3)
        t = time.perf_counter()
        arena.py_vs_py(_Eng("trainee", 2.0), _Eng("baseline", 0.5), (10000, 0x5EED), max(args.games // 4, 1))
        play_s = time.perf_counter() - t
        games, paths = arena.last_games, list(arena.last_log_paths)
        make_files, make_games = _iters(games, paths, grp, args)
        n_batches = check_equal(make_files, make_games, 99)
        times = {"files": [], "games": []}
        samples = {}
        for r in range(args.rounds):
            for name, make in (("files", make_files), ("games", make_games)):
                s, n = run_arm(make, 100 + r)
                times[name].append(s)
                samples[name] = n
        conv = converter_ms(games)
    med = {k: statistics.median(v) for k, v in times.items()}
    print(json.dumps({"gpu": gpu, "games": len(games), "play_s": round(play_s, 3), "batches": n_batches, "equal": True,
                      "samples_per_pass": samples["games"],
                      "files_s": med["files"], "games_s": med["games"], "files_samples_per_s": samples["files"] / med["files"],
                      "games_samples_per_s": samples["games"] / med["games"], "files_over_games": med["files"] / med["games"],
                      "converter_ms_all_games": conv, "rounds": {k: [round(x, 4) for x in v] for k, v in times.items()}}))


if __name__ == "__main__":
    main()
