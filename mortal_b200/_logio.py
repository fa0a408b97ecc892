"""Reading log files for the device decoder (csrc/mjx_mjai.cuh), shared by stat.Stat.from_dir, dataset.GameplayLoader, dataset.Grp
and the validate_logs CLI: when the device path may run, the files' raw bytes are read on a thread pool in chunks of consecutive
files bounded by count and text size, staged once into pinned memory, copied to the device and gunzipped there straight into the
text buffer the decoder reads (k_gunzip, csrc/mjx_inflate.cuh; plain files are copied into the same buffer). A file the device
cannot take (unreadable, too short to be a gzip member, an ISIZE no deflate stream of its length can reach, or declined by
k_gunzip) goes back to the caller's host code, which reads it as before."""
from __future__ import annotations

import gzip
import locale
import os

import numpy as np

from . import _cdecl

# the device paths decode and reduce the files in chunks of consecutive files: at most CHUNK_LOGS files and, unless a single file
# is larger, CHUNK_BYTES of decompressed text. A chunk's compressed bytes are held three times (the file contents, the pinned
# staging buffer, the device copy) and its text once, on the device, so this bounds memory whatever the corpus size.
CHUNK_LOGS = 4096
CHUNK_BYTES = 256 << 20
GZ_MIN_BYTES = 18   # a gzip member's 10-byte header and 8-byte trailer
GZ_MAX_RATIO = 1032  # DEFLATE's largest expansion: a 258-byte match in 2 bits (RFC 1951), with the header and trailer on top
# k_gunzip runs one warp per file, so a launch lasts as long as its slowest file (about 70 ms for a 530 KB arena log on an H100):
# a batch of fewer gzip files than this is gunzipped on the thread pool instead (DESIGN.md §5: a 20-file loader batch is faster
# there, 1,024 files are faster on the device)
GZ_DEVICE_MIN_FILES = 64

HEADER = os.path.join(os.path.dirname(_cdecl.HEADER), "mjx_logio.h")
with open(HEADER) as _f:
    _TEXT = _f.read()
SYMBOLS = _cdecl.functions(_TEXT, "mjx_")  # the entries of include/mjx_logio.h, exported by libmjx.so
GUNZIP_STATUSES = tuple(name for _, name in _cdecl.xmacro(_TEXT, "MJX_GUNZIP_STATUSES"))  # indexed by k_gunzip's status code
_BOUND = None


def _load():
    global _BOUND
    if _BOUND is None:
        from . import _lib

        _BOUND = _cdecl.bind(_lib.load(), SYMBOLS)
    return _BOUND


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


def chunks(paths, pool, step: int, read=read_bytes, max_logs: int = CHUNK_LOGS, max_bytes: int = CHUNK_BYTES, size=len):
    """(paths, contents) of consecutive files in order, read by `read` on `pool` `step` at a time, cut at max_logs files or max_bytes
    of text, a file's text being size(content) (a chunk always takes at least one file)"""
    cur, size_, lo = [], 0, 0
    for s in range(0, len(paths), step):
        for b in pool.map(read, paths[s:s + step]):
            n = size(b) if b is not None else 0
            if cur and (len(cur) >= max_logs or size_ + n > max_bytes):
                yield paths[lo:lo + len(cur)], cur
                lo += len(cur); cur, size_ = [], 0
            cur.append(b); size_ += n
    if cur:
        yield paths[lo:lo + len(cur)], cur


def read_file(path: str, gz: bool | None = None):
    """(the file's raw bytes or None when they cannot be read, whether it is read as gzip: default for a `.gz` name); the device
    gunzips it (stage)"""
    gz = path.lower().endswith(".gz") if gz is None else gz
    try:
        with open(path, "rb") as f:
            return f.read(), gz
    except Exception:  # noqa: BLE001 — any failure: the host path raises its own exception for this file
        return None, gz


def read_gz_file(path: str):
    """read_file of a file every loader opens with gzip.open, whatever its name"""
    return read_file(path, True)


def gz_isize(raw: bytes):
    """the text size a gzip member's trailer states (its last four bytes), or None when the device does not take the file: shorter
    than a header and trailer, or a size beyond what DEFLATE can expand its bytes to"""
    if len(raw) < GZ_MIN_BYTES:
        return None
    n = int.from_bytes(raw[-4:], "little")
    return n if n <= GZ_MAX_RATIO * len(raw) else None


def text_size(item) -> int:
    """the device text a read_file item takes: its ISIZE, its length for a plain file, 0 for a file left to the host"""
    raw, gz = item
    if raw is None:
        return 0
    return (gz_isize(raw) or 0) if gz else len(raw)


class DeviceText:
    """The texts of a chunk of files on the device, one slot per file taken: slot j is file files[j], its text
    text[log_off[j], log_off[j + 1]) (a uint8 tensor); status int32 [m] on the device is its k_gunzip status (0 for a plain
    file). The gzip slots come first, so one k_gunzip launch covers them."""

    def __init__(self, text, log_off, status, files):
        self.text, self.log_off, self.status, self.files = text, log_off, status, files


def _host_gunzip(item):
    raw, gz = item
    if not gz or raw is None:
        return item
    try:
        return gzip.decompress(raw), False
    except Exception:  # noqa: BLE001 — any failure: the host path raises its own exception for this file
        return None, False


def stage(items, device: int, pool=None) -> DeviceText:
    """read_file items -> DeviceText on `device`: the bytes of every file taken copied once into pinned memory and once to the
    device, the gzip ones inflated there by mjx_gunzip_dev, the plain ones copied into the same buffer; enqueued on the current
    stream without a synchronise (the status says which gzip files were declined). With fewer than GZ_DEVICE_MIN_FILES gzip
    files, `pool` gunzips them and their texts are copied as plain files."""
    import torch

    from . import _lib

    if pool is not None and sum(1 for raw, z in items if z and raw is not None) < GZ_DEVICE_MIN_FILES:
        items = list(pool.map(_host_gunzip, items))
    gz = [k for k, (raw, z) in enumerate(items) if z and raw is not None and gz_isize(raw) is not None]
    plain = [k for k, (raw, z) in enumerate(items) if not z and raw is not None]
    files = gz + plain
    raws = [items[k][0] for k in files]
    m = len(files)
    in_off = np.zeros(m + 1, dtype=np.int64)
    np.cumsum([len(b) for b in raws], out=in_off[1:])
    log_off = np.zeros(m + 1, dtype=np.int64)
    np.cumsum([gz_isize(b) for b in raws[:len(gz)]] + [len(b) for b in raws[len(gz):]], out=log_off[1:])
    dev = torch.device("cuda", device)
    staged = torch.empty(max(int(in_off[-1]), 1), dtype=torch.uint8, pin_memory=True)
    view = staged.numpy()
    for b, o in zip(raws, in_off):
        view[o:o + len(b)] = np.frombuffer(b, dtype=np.uint8)
    # non_blocking: `staged` must outlive the copy; the callers' first copy back synchronises the stream before it is freed
    d_in = staged.to(dev, non_blocking=True)
    text = torch.empty(max(int(log_off[-1]), 1), dtype=torch.uint8, device=dev)
    status = torch.zeros(m, dtype=torch.int32, device=dev)
    g = len(gz)
    if g:
        offs = torch.from_numpy(np.concatenate([in_off[:g + 1], log_off[:g + 1]])).to(dev)
        _lib.check(_load().mjx_gunzip_dev(g, d_in.data_ptr(), int(in_off[g]), offs.data_ptr(), text.data_ptr(), int(log_off[g]),
                                          offs[g + 1:].data_ptr(), status.data_ptr(), torch.cuda.current_stream(dev).cuda_stream),
                   "mjx_gunzip_dev")
    if m > g:
        text[int(log_off[g]):int(log_off[m])].copy_(d_in[int(in_off[g]):int(in_off[m])])
    out = DeviceText(text, log_off, status, files)
    out._keep = (staged, d_in)
    return out


def count_keys(text, log_off, keys, device: int) -> np.ndarray:
    """bytes.count of every key over every log text[log_off[j], log_off[j + 1]) on the device -> int64 [n_logs, len(keys)]"""
    import torch

    from . import _lib

    n = len(log_off) - 1
    koff = np.zeros(len(keys) + 1, dtype=np.int32)
    np.cumsum([len(k) for k in keys], out=koff[1:])
    kb = np.frombuffer(b"".join(keys), dtype=np.uint8).copy()
    dev = torch.device("cuda", device)
    out = torch.empty((n, len(keys)), dtype=torch.int64, device=dev)
    if n == 0:
        return np.zeros((0, len(keys)), dtype=np.int64)
    d_off = torch.from_numpy(np.ascontiguousarray(log_off, dtype=np.int64)).to(dev)
    _lib.check(_load().mjx_count_keys_dev(n, text.data_ptr(), text.numel(), d_off.data_ptr(), kb.ctypes.data, koff.ctypes.data,
                                          len(keys), out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream),
               "mjx_count_keys_dev")
    return out.cpu().numpy()


def spans(text, log_off, idx, begin, end, device: int):
    """the bytes [begin[k], end[k]) of log idx[k] of text (offsets relative to the log), gathered on the device and copied back
    once -> list of bytes"""
    import torch

    if not len(idx):
        return []
    dev = torch.device("cuda", device)
    lo = np.asarray(log_off, dtype=np.int64)[np.asarray(idx, dtype=np.int64)] + np.asarray(begin, dtype=np.int64)
    ln = np.asarray(end, dtype=np.int64) - np.asarray(begin, dtype=np.int64)
    cut = np.zeros(len(ln) + 1, dtype=np.int64)
    np.cumsum(ln, out=cut[1:])
    d_lo = torch.from_numpy(lo).to(dev)
    d_ln = torch.from_numpy(ln).to(dev)
    at = torch.repeat_interleave(d_lo - torch.from_numpy(cut[:-1]).to(dev), d_ln, output_size=int(cut[-1]))
    at += torch.arange(int(cut[-1]), device=dev)
    flat = text[at].cpu().numpy().tobytes()
    return [flat[cut[k]:cut[k + 1]] for k in range(len(ln))]
