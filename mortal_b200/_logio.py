"""Reading log files for the device decoder (csrc/mjx_mjai.cuh), shared by stat.Stat.from_dir, dataset.GameplayLoader and
dataset.Grp: when the device path may run, the files' bytes read and gunzipped on a thread pool, and chunks of consecutive files
bounded by count and size. A file the device cannot take goes back to the caller's host code, which reads it as before."""
from __future__ import annotations

import gzip
import locale
import os

# the device paths decode and reduce the files in chunks of consecutive files: at most CHUNK_LOGS files and, unless a single file
# is larger, CHUNK_BYTES of decompressed text. The text of a chunk is held three times (the file contents, the pinned staging
# buffer, the device copy), so this bounds memory whatever the corpus size.
CHUNK_LOGS = 4096
CHUNK_BYTES = 256 << 20


def device_ready() -> bool:
    """the device path needs the built library, a CUDA device, and a UTF-8 locale (the host path reads the files in the locale's
    encoding; the decoder reads UTF-8)"""
    from . import _lib

    if not os.path.exists(_lib.lib_path()) or locale.getpreferredencoding(False).lower().replace("-", "") != "utf8":
        return False
    try:
        import torch
    except ImportError:
        return False
    return torch.cuda.is_available()


def log_device() -> int:
    """the GPU the log readers run on: the one libmjx is initialised on (the library serves one device per process, so a process
    whose arena or engine lives on cuda:k reads its logs there too), else torch's current device"""
    from . import _lib

    if _lib._INIT_DEVICE is not None:
        return _lib._INIT_DEVICE
    import torch

    return torch.cuda.current_device()


def read_bytes(path: str, gz: bool | None = None):
    """a file's bytes, gunzipped when `gz` (default: for a `.gz` name); None when that fails (the host path then decides)"""
    try:
        if path.lower().endswith(".gz") if gz is None else gz:
            with gzip.open(path, "rb") as f:
                return f.read()
        with open(path, "rb") as f:
            return f.read()
    except Exception:  # noqa: BLE001 — any failure: the host path raises its own exception for this file
        return None


def read_gz(path: str):
    """read_bytes of a file every reader opens with gzip.open, whatever its name"""
    return read_bytes(path, True)


def utf8_ok(blob: bytes) -> bool:
    """whether the text reader of a UTF-8 locale decodes `blob` without an error"""
    if blob.isascii():
        return True
    try:
        blob.decode("utf-8")
    except UnicodeDecodeError:
        return False
    return True


def host_text(blob: bytes) -> str:
    """the str that open(..., "rt") in a UTF-8 locale returns for `blob`: UTF-8, universal newlines"""
    return blob.decode("utf-8").replace("\r\n", "\n").replace("\r", "\n")


def chunks(paths, pool, step: int, read=read_bytes, max_logs: int = CHUNK_LOGS, max_bytes: int = CHUNK_BYTES):
    """(paths, contents) of consecutive files in order, read by `read` on `pool` `step` at a time, cut at max_logs files or max_bytes
    of text (a chunk always takes at least one file)"""
    cur, size, lo = [], 0, 0
    for s in range(0, len(paths), step):
        for b in pool.map(read, paths[s:s + step]):
            n = len(b) if b is not None else 0
            if cur and (len(cur) >= max_logs or size + n > max_bytes):
                yield paths[lo:lo + len(cur)], cur
                lo += len(cur); cur, size = [], 0
            cur.append(b); size += n
    if cur:
        yield paths[lo:lo + len(cur)], cur
