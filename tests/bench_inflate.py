#!/usr/bin/env python
"""Gunzip on the host against gunzip on the device (k_gunzip, csrc/mjx_inflate.cuh), both arms alternated in one process over
arena logs generated in the run:

  * read + gunzip: thread-pool gzip against thread-pool raw reads + mjx_gunzip_dev (wall clock to the device text), with the
    kernel alone timed by CUDA events and the bytes each arm copies host to device;
  * end to end at all files: the validate_logs CLI, Stat.from_dir and Grp.load_gz_log_files;
  * GameplayLoader.load_gz_log_files per --batch-file batch (the trainer's file_batch_size).

The host arm is the readers' previous data path: _logio's readers patched to gunzip on the thread pool and hand the text to the
device as a plain file (and, for the CLI, _read on the pool then _validate). The outputs of the two arms are checked equal, and
every arena log must be accepted by the kernel. Prints the GPU name and power limit beside the numbers."""
import argparse
import contextlib
import glob
import io
import os
import statistics
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from mortal_b200 import _lib, _logio, validate_logs  # noqa: E402
from mortal_b200.dataset import GameplayLoader, Grp  # noqa: E402
from mortal_b200.libriichi.arena import OneVsThree  # noqa: E402
from mortal_b200.stat import Stat  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--games", type=int, default=1024, help="arena games (a multiple of 4)")
ap.add_argument("--batch", type=int, default=20, help="files per GameplayLoader.load_gz_log_files call")
ap.add_argument("--batches", type=int, default=10, help="loader calls timed per arm")
ap.add_argument("--rounds", type=int, default=3, help="alternated rounds of the end-to-end readers")
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


@contextlib.contextmanager
def host_gunzip():
    """the previous read path: gunzip on the thread pool, the text staged and copied as a plain file"""
    rf, rg = _logio.read_file, _logio.read_gz_file
    _logio.read_file = lambda p, gz=None: (_logio.read_bytes(p, gz), False)
    _logio.read_gz_file = lambda p: (_logio.read_gz(p), False)
    try:
        yield
    finally:
        _logio.read_file, _logio.read_gz_file = rf, rg


@contextlib.contextmanager
def device_gunzip():
    """k_gunzip for every batch, however few files it has"""
    keep = _logio.GZ_DEVICE_MIN_FILES
    _logio.GZ_DEVICE_MIN_FILES = 0
    try:
        yield
    finally:
        _logio.GZ_DEVICE_MIN_FILES = keep


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def cli_device(d):
    with contextlib.redirect_stdout(io.StringIO()) as buf:
        validate_logs.main([d])
    return buf.getvalue()


def cli_host(d):  # the CLI's previous loop: _read (host gunzip) on the pool, then _validate
    paths = sorted(set(glob.glob(os.path.join(d, "**", "*.json"), recursive=True))
                   | set(glob.glob(os.path.join(d, "**", "*.json.gz"), recursive=True)))
    out = []
    with ThreadPoolExecutor(min(32, os.cpu_count() or 1)) as pool:
        for lo in range(0, len(paths), validate_logs.CHUNK_LOGS):
            chunk = paths[lo:lo + validate_logs.CHUNK_LOGS]
            verdicts, enc = validate_logs._validate(list(pool.map(validate_logs._read, chunk)))
            out += [f"\nerror in log {p}\n{validate_logs.message(v, e)}\n" for p, v, e in zip(chunk, verdicts, enc) if v is not None]
    return "".join(out)


def main():
    assert _logio.device_ready(), "the device path needs libmjx, a CUDA device and a UTF-8 locale"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(f"GPU: {torch.cuda.get_device_name(0)} | nvidia-smi: {smi[0] if smi else 'n/a'}")
    _lib.init(0)
    with tempfile.TemporaryDirectory() as d:
        torch.manual_seed(0)
        OneVsThree(disable_progress_bar=True, log_dir=d).py_vs_py(Eng("alpha"), Eng("beta"), (77000, 13), args.games // 4)
        files = sorted(glob.glob(os.path.join(d, "*.json.gz")))
        raws = [open(f, "rb").read() for f in files]
        n_gz, n_text = sum(len(b) for b in raws), sum(_logio.gz_isize(b) for b in raws)
        print(f"{len(files)} arena logs: {n_gz / 1e6:.1f} MB gzipped, {n_text / 1e6:.1f} MB of text")

        # every arena log is accepted, and its text is Python's
        T = _logio.stage([(b, True) for b in raws], 0)
        st = T.status.cpu().numpy()
        assert len(T.files) == len(files) and (st == 0).all(), np.bincount(st)
        text = T.text.cpu().numpy().tobytes()
        import gzip

        for j, k in enumerate(T.files[:64]):
            assert text[T.log_off[j]:T.log_off[j + 1]] == gzip.decompress(raws[k])
        print("every arena log accepted by k_gunzip; texts equal gzip.decompress")

        # the kernel alone, on device-resident bytes (CUDA events)
        dev = torch.device("cuda", 0)
        gz = torch.from_numpy(np.frombuffer(b"".join(raws), dtype=np.uint8).copy()).to(dev)
        in_off = np.zeros(len(raws) + 1, dtype=np.int64); np.cumsum([len(b) for b in raws], out=in_off[1:])
        out_off = np.asarray(T.log_off, dtype=np.int64)
        L = _logio._load()
        stream = torch.cuda.current_stream(dev).cuda_stream

        def kernel(n):
            offs = torch.from_numpy(np.concatenate([in_off[:n + 1], out_off[:n + 1]])).to(dev)
            status = torch.empty(n, dtype=torch.int32, device=dev)
            out = torch.empty(int(out_off[n]), dtype=torch.uint8, device=dev)
            for _ in range(3):
                L.mjx_gunzip_dev(n, gz.data_ptr(), int(in_off[n]), offs.data_ptr(), out.data_ptr(), int(out_off[n]),
                                 offs[n + 1:].data_ptr(), status.data_ptr(), stream)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                L.mjx_gunzip_dev(n, gz.data_ptr(), int(in_off[n]), offs.data_ptr(), out.data_ptr(), int(out_off[n]),
                                 offs[n + 1:].data_ptr(), status.data_ptr(), stream)
            e1.record()
            torch.cuda.synchronize()
            assert (status == 0).all()
            return e0.elapsed_time(e1) / args.reps

        k_all, k_batch = kernel(len(raws)), kernel(args.batch)
        print(f"k_gunzip alone: {k_all:.2f} ms for {len(raws)} files ({n_text / k_all / 1e6:.1f} GB/s of text), "
              f"{k_batch:.2f} ms for {args.batch} files")

        # read + gunzip to the device text: thread-pool gzip + text H2D against raw reads + gz H2D + k_gunzip, alternated
        workers = min(32, os.cpu_count() or 1)
        t_host, t_dev = [], []
        with ThreadPoolExecutor(workers) as pool:
            for _ in range(args.rounds + 1):
                dt, _ = timed(lambda: _logio.stage(list(pool.map(lambda p: (_logio.read_gz(p), False), files)), 0).text)
                t_host.append(dt)
                dt, _ = timed(lambda: _logio.stage(list(pool.map(_logio.read_gz_file, files)), 0).text)
                t_dev.append(dt)
        med = lambda xs: statistics.median(xs[1:])  # the first round warms up
        print(f"read + gunzip to device text, {len(files)} files: thread-pool gzip {med(t_host) * 1e3:.1f} ms "
              f"(H2D {n_text / 1e6:.1f} MB) | device {med(t_dev) * 1e3:.1f} ms (H2D {n_gz / 1e6:.1f} MB)")

        # end to end, alternated; the arms' results must be equal
        for name, dev_fn, host_fn, same in (
                ("validate_logs CLI", lambda: cli_device(d), lambda: cli_host(d), lambda a, b: a == b),
                ("Stat.from_dir", lambda: repr(Stat.from_dir(d, "alpha")), None, lambda a, b: a == b),
                ("Grp.load_gz_log_files", lambda: Grp.load_gz_log_files(files), None,
                 lambda a, b: all(np.array_equal(x.take_feature(), y.take_feature()) and x.take_rank_by_player() == y.take_rank_by_player()
                                  for x, y in zip(a, b)))):
            th, td = [], []
            for _ in range(args.rounds + 1):
                if host_fn is None:
                    with host_gunzip():
                        dt, a = timed(dev_fn)
                else:
                    dt, a = timed(host_fn)
                th.append(dt)
                with device_gunzip():
                    dt, b = timed(dev_fn)
                td.append(dt)
                assert same(a, b), name
            print(f"{name}, {len(files)} files: host gunzip {med(th):.3f} s | device gunzip {med(td):.3f} s "
                  f"({med(th) / med(td):.2f}x)")

        # GameplayLoader per batch of files
        loader = GameplayLoader(4, oracle=False)
        batches = [files[k * args.batch:(k + 1) * args.batch] for k in range(args.batches + 1)]
        th, td, ts = [], [], []
        for b in batches:
            with host_gunzip():
                dt, a = timed(lambda: loader.load_gz_log_files(b))
            th.append(dt)
            with device_gunzip():
                dt, c = timed(lambda: loader.load_gz_log_files(b))
            td.append(dt)
            dt, e = timed(lambda: loader.load_gz_log_files(b))
            ts.append(dt)
            for r in (c, e):
                assert all(torch.equal(x.take_obs(), y.take_obs()) for pa, pc in zip(a, r) for x, y in zip(pa, pc))
        print(f"GameplayLoader.load_gz_log_files, {args.batch}-file batches: host gunzip {med(th) * 1e3:.1f} ms | "
              f"device gunzip {med(td) * 1e3:.1f} ms | as selected ({args.batch} < {_logio.GZ_DEVICE_MIN_FILES} files: "
              f"{'pool' if args.batch < _logio.GZ_DEVICE_MIN_FILES else 'device'}) {med(ts) * 1e3:.1f} ms per batch")


if __name__ == "__main__":
    main()
