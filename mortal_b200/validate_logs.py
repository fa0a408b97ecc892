"""libriichi bin/validate_logs.rs on the GPU: replay mjai logs through the four seats and report the first move a rule forbids.

    validate_logs(texts) -> [Verdict | None]      (None = the log is valid; all logs of a call run in one launch)
    python -m mortal_b200.validate_logs DIR       (every DIR/**/*.json and DIR/**/*.json.gz, in sorted order)

The log text is decoded into event words on the device (k_mjai_decode, csrc/mjx_mjai.cuh), and the words go straight to the
k_validate_logs kernel (csrc/mjx_validate.cuh), which runs the rule checks and the state updates. A log the device decoder
declines (anything it cannot show Python's json reads the same way, and every log that fails to parse) is decoded on the host
by encode_log (json.loads + dataset_codec.check_event, reported as PARSE) exactly as before; the verdicts do not depend on the
path. There is no CPU path: without a CUDA device validate_logs raises.
"""
from __future__ import annotations

import glob
import gzip
import json
import os
import sys
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass

import numpy as np

from . import _cdecl, _lib
from .dataset_codec import HORA_WORDS, KYOKU_WORDS, check_event, encode_events

# indexed by code, read from include/mjx.h (their single definition): the verdict status names (mjx_verdict_status, whose codes
# run 0, 1, ...) and the reason names (MJX_VALIDATE_REASONS)
STATUSES = tuple(name.removeprefix("MJX_V_") for name in _cdecl.enum(_cdecl.header(), "mjx_verdict_status"))
REASONS = tuple(name for _, name in _cdecl.xmacro(_cdecl.header(), "MJX_VALIDATE_REASONS"))
CHUNK_LOGS = 4096  # logs decoded and validated per launch by the CLI: bounds its memory whatever the corpus size


@dataclass(frozen=True)
class Verdict:
    status: str  # one of STATUSES other than OK
    reason: str  # one of REASONS
    line: int    # 1-based line of the offending event
    seat: int    # UPDATE: the lowest seat whose update fails; CHECK: the actor; else -1


@dataclass
class EncodedLog:
    hdr: np.ndarray    # uint64 [n] event words
    kyoku: np.ndarray  # uint64 [k, KYOKU_WORDS] start_kyoku payloads
    hora: np.ndarray   # uint64 [h, HORA_WORDS] hora side entries
    lines: list        # line number of every event
    texts: list        # the event lines themselves


def encode_log(text: str):
    """One log -> EncodedLog, or the Verdict of a host-side rejection (PARSE, or UNSUPPORTED for a start_kyoku whose round
    wind is not a wind). The whole log is parsed before anything is replayed, as the reference does."""
    events, lines, raw = [], [], []
    for no, ln in enumerate(text.splitlines(), 1):
        if not ln.strip():
            continue
        try:
            ev = json.loads(ln)
        except ValueError:
            return Verdict("PARSE", "json", no, -1)
        why = check_event(ev)
        if why is not None:
            return Verdict("PARSE", why, no, -1)
        if ev["type"] == "start_kyoku" and ev["bakaze"] not in ("E", "S", "W", "N"):
            return Verdict("UNSUPPORTED", "capacity", no, -1)
        events.append(ev); lines.append(no); raw.append(ln)
    hora = []
    hdr, pay = encode_events(events, hora=hora)
    return EncodedLog(hdr, pay, np.array(hora, dtype=np.uint64).reshape(-1, HORA_WORDS), lines, raw)


def pack(encoded):
    """EncodedLogs -> the concatenated host arrays mjx_validate_logs takes (the build_jobs layout plus the hora side array)"""
    n = len(encoded)
    ev_off, ev_cnt, ky_off, ho_off = (np.zeros(n, dtype=np.int32) for _ in range(4))
    nh = nk = no = 0
    for i, e in enumerate(encoded):
        ev_off[i], ev_cnt[i], ky_off[i], ho_off[i] = nh, len(e.hdr), nk, no
        nh += len(e.hdr); nk += len(e.kyoku); no += len(e.hora)
    cat = lambda xs, w: np.ascontiguousarray(np.concatenate(xs).reshape(-1) if xs else np.zeros(w, dtype=np.uint64), dtype=np.uint64)
    return dict(hdr=cat([e.hdr for e in encoded], 0), ev_off=ev_off, ev_cnt=ev_cnt, kyoku=cat([e.kyoku for e in encoded], 0),
                ky_off=ky_off, hora=cat([e.hora for e in encoded], 0), hora_off=ho_off)


def run_packed(p, device: int = 0) -> np.ndarray:
    """mjx_validate_logs over pack()'s arrays -> int32 [n, 4] (status, reason, event index + 1, seat)"""
    L = _lib.load()
    _lib.init(device)
    n = len(p["ev_off"])
    out = np.zeros((n, 4), dtype=np.int32)
    if n == 0:
        return out
    _lib.check(L.mjx_validate_logs(n, p["hdr"].ctypes.data, p["ev_off"].ctypes.data, p["ev_cnt"].ctypes.data, len(p["hdr"]),
                                   p["kyoku"].ctypes.data, p["ky_off"].ctypes.data, len(p["kyoku"]), p["hora"].ctypes.data,
                                   p["hora_off"].ctypes.data, len(p["hora"]), out.ctypes.data, None), "mjx_validate_logs")
    return out


def to_verdict(row, e: EncodedLog):
    status, reason, idx, seat = (int(x) for x in row)
    if status == 0:
        return None
    return Verdict(STATUSES[status], REASONS[reason], e.lines[idx - 1] if 0 < idx <= len(e.lines) else idx, seat)


@dataclass
class DecodedLogs:
    """mjx_mjai_count_dev + mjx_mjai_fill_dev over a batch of texts: per-log counts on the host, the arrays on the device
    (torch tensors, validate_logs.pack() layout; a declined log has no entries and ev_cnt 0)."""
    accept: np.ndarray  # bool [n]
    counts: np.ndarray  # int32 [n, 6] mjx_mjai_counts
    ev_off: np.ndarray; ev_cnt: np.ndarray; ky_off: np.ndarray; hora_off: np.ndarray  # int32 [n]
    offs: object        # int32 [4, n] device: ev_off, ev_cnt, ky_off, hora_off
    hdr: object         # int64 [n_events] device (the uint64 words)
    lines: object       # int32 [n_events] device: 1-based line of every event
    kyoku: object       # int64 [n_kyoku * KYOKU_WORDS] device
    hora: object        # int64 [n_hora * HORA_WORDS] device
    deltas: object = None      # with deltas=True: int32 [n_events, 4] device, every hora's and ryukyoku's deltas at its event
    has_deltas: object = None  # with deltas=True: uint8 [n_events] device, 1 where that event's `deltas` is present and not null


def decode_dev(blobs, device: int = 0, augment: bool = False, deltas: bool = False) -> DecodedLogs:
    """UTF-8 log texts (bytes) -> DecodedLogs, decoded on `device` (csrc/mjx_mjai.cuh); the one device-to-host copy is the counts.
    `deltas` also fills the per-event deltas arrays (mjx_mjai_fill_deltas_dev); the other arrays are the same either way."""
    import torch

    L = _lib.load()
    n = len(blobs)
    dev = torch.device("cuda", device)
    st = torch.cuda.current_stream(dev).cuda_stream
    log_off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(b) for b in blobs], out=log_off[1:])
    staged = torch.empty(max(int(log_off[-1]), 1), dtype=torch.uint8, pin_memory=True)  # the texts copied once, into pinned memory
    view = staged.numpy()
    for b, o in zip(blobs, log_off):
        view[o:o + len(b)] = np.frombuffer(b, dtype=np.uint8)
    text = staged.to(dev, non_blocking=True)  # `staged` lives until the counts' copy below has synchronised the stream
    d_off = torch.from_numpy(log_off).to(dev)
    d_counts = torch.empty((n, 6), dtype=torch.int32, device=dev)
    _lib.check(L.mjx_mjai_count_dev(n, text.data_ptr(), int(log_off[-1]), d_off.data_ptr(), int(augment), d_counts.data_ptr(), st),
               "mjx_mjai_count_dev")
    counts = d_counts.cpu().numpy()
    accept = counts[:, 0] != 0
    excl = lambda x: (np.cumsum(x) - x).astype(np.int32)
    ev_cnt, n_ky, n_ho = (counts[:, k].astype(np.int32) for k in (1, 2, 3))
    ev_off, ky_off, hora_off = excl(ev_cnt), excl(n_ky), excl(n_ho)
    n_ev, n_k, n_h = int(ev_cnt.sum()), int(n_ky.sum()), int(n_ho.sum())
    offs = torch.from_numpy(np.stack([ev_off, ev_cnt, ky_off, hora_off])).to(dev)
    hdr = torch.empty(n_ev, dtype=torch.int64, device=dev)
    lines = torch.empty(n_ev, dtype=torch.int32, device=dev)
    kyoku = torch.empty(n_k * KYOKU_WORDS, dtype=torch.int64, device=dev)
    hora = torch.empty(n_h * HORA_WORDS, dtype=torch.int64, device=dev)
    ptr = lambda t: t.data_ptr() if t.numel() else None
    if deltas:
        d_deltas = torch.empty((n_ev, 4), dtype=torch.int32, device=dev)
        d_has = torch.empty(n_ev, dtype=torch.uint8, device=dev)
        if accept.any():
            _lib.check(L.mjx_mjai_fill_deltas_dev(n, text.data_ptr(), int(log_off[-1]), d_off.data_ptr(), int(augment),
                                                  d_counts.data_ptr(), offs[0].data_ptr(), offs[2].data_ptr(), offs[3].data_ptr(),
                                                  ptr(hdr), ptr(lines), n_ev, ptr(kyoku), n_k * KYOKU_WORDS, ptr(hora),
                                                  n_h * HORA_WORDS, ptr(d_deltas), ptr(d_has), st), "mjx_mjai_fill_deltas_dev")
        return DecodedLogs(accept, counts, ev_off, ev_cnt, ky_off, hora_off, offs, hdr, lines, kyoku, hora, d_deltas, d_has)
    if accept.any():
        _lib.check(L.mjx_mjai_fill_dev(n, text.data_ptr(), int(log_off[-1]), d_off.data_ptr(), int(augment), d_counts.data_ptr(),
                                       offs[0].data_ptr(), offs[2].data_ptr(), offs[3].data_ptr(), ptr(hdr), ptr(lines), n_ev,
                                       ptr(kyoku), n_k * KYOKU_WORDS, ptr(hora), n_h * HORA_WORDS, st), "mjx_mjai_fill_dev")
    return DecodedLogs(accept, counts, ev_off, ev_cnt, ky_off, hora_off, offs, hdr, lines, kyoku, hora)


@dataclass
class _Lines:
    lines: list  # line number of every event
    texts: list  # the event lines themselves


def _event_lines(text: str) -> _Lines:
    """the lines and line numbers of a log's events, for message(): every non-blank line of a log the device accepted is an event"""
    nos, raw = [], []
    for no, ln in enumerate(text.splitlines(), 1):
        if ln.strip():
            nos.append(no); raw.append(ln)
    return _Lines(nos, raw)


def _validate(texts, device: int = 0):
    """-> ([Verdict | None], per log the EncodedLog / line list message() reads, or None for a valid log decoded on the device).
    Logs are decoded on the device; those it declines go through encode_log, as do texts that are not valid UTF-8."""
    import torch

    _lib.init(device)  # no CUDA device: raises before any work, whatever the logs
    L = _lib.load()
    out, enc = [None] * len(texts), [None] * len(texts)
    blobs, idx, host = [], [], []  # host: the logs encode_log decodes
    for i, t in enumerate(texts):
        if isinstance(t, Verdict):
            out[i] = enc[i] = t
            continue
        try:
            blobs.append(t.encode("utf-8")); idx.append(i)
        except UnicodeEncodeError:  # lone surrogates: not UTF-8, so the host decides
            host.append(i)
    if blobs:
        D = decode_dev(blobs, device)
        n = len(blobs)
        dev = torch.device("cuda", device)
        verd = torch.empty((n, 4), dtype=torch.int32, device=dev)
        ptr = lambda t: t.data_ptr() if t.numel() else None
        _lib.check(L.mjx_validate_logs_dev(n, ptr(D.hdr), D.offs[0].data_ptr(), D.offs[1].data_ptr(), D.hdr.numel(), ptr(D.kyoku),
                                           D.offs[2].data_ptr(), D.kyoku.numel(), ptr(D.hora), D.offs[3].data_ptr(), D.hora.numel(),
                                           verd.data_ptr(), torch.cuda.current_stream(dev).cuda_stream), "mjx_validate_logs_dev")
        rows = verd.cpu().numpy()
        bad = np.nonzero(D.accept & (rows[:, 0] != 0))[0]
        ev = rows[bad, 2].astype(np.int64)
        inside = (ev > 0) & (ev <= D.ev_cnt[bad])
        lines = np.array(ev)
        if inside.any():  # the line of the failing event, from the device line array
            at = torch.from_numpy(D.ev_off[bad][inside].astype(np.int64) + ev[inside] - 1).to(dev)
            lines[inside] = D.lines[at].cpu().numpy()
        for k, b in enumerate(bad):
            status, reason, _, seat = (int(x) for x in rows[b])
            out[idx[b]] = Verdict(STATUSES[status], REASONS[reason], int(lines[k]), seat)
            enc[idx[b]] = _event_lines(texts[idx[b]])
        host += [idx[k] for k in np.nonzero(~D.accept)[0]]
    for i in host:
        enc[i] = encode_log(texts[i])
        if isinstance(enc[i], Verdict):
            out[i] = enc[i]
    replay = [i for i in host if isinstance(enc[i], EncodedLog)]
    if replay:
        rows = run_packed(pack([enc[i] for i in replay]), device)
        for i, r in zip(replay, rows):
            out[i] = to_verdict(r, enc[i])
    return out, enc


def validate_logs(texts, device: int = 0):
    """bin/validate_logs.rs process_path over every text (one mjai event per line) -> [Verdict | None]; one kernel launch."""
    return _validate(texts, device)[0]


_CHECK_TEXT = {"chi from non-kamicha": "chi from non-kamicha at line {line}", "missing ura_markers": "missing field `ura_markers`",
               "missing deltas": "missing field `deltas`", "agari_points": "failed to get agari points at line {line}",
               "deltas below points": "deltas[actor] < agari points (rough test) at line {line}"}


def message(v: Verdict, e) -> str:
    """the reference's report of a failure: what failed at which line, the event, and the seat's brief_info() before it"""
    if v.status == "CHECK":
        head = _CHECK_TEXT.get(v.reason, "fails {reason} at line {line}").format(reason=v.reason, line=v.line)
    elif v.status == "UPDATE":
        head = f"fails update of seat {v.seat} ({v.reason}) at line {v.line}"
    elif v.status == "PARSE":
        return f"fails to parse ({v.reason}) at line {v.line}"
    else:
        return f"unsupported event at line {v.line}: this implementation's table record cannot hold it"
    idx = e.lines.index(v.line)
    return f"{head}\naction: {e.texts[idx]}\nstate:\n{_brief_info(e.texts[:idx], v.seat)}"


def _brief_info(prefix, seat: int) -> str:
    """PlayerState::brief_info of `seat` after the events before the failing one (only failing logs pay for this replay)"""
    from .libriichi.state import PlayerState

    ps = PlayerState(seat)
    for ln in prefix:
        ps.update(ln)
    return ps.brief_info()


def _read(path: str):
    """the text of a log, or a PARSE verdict when it cannot be read or decoded"""
    try:
        if path.lower().endswith(".gz"):
            with gzip.open(path, "rt", encoding="utf-8") as f:
                return f.read()
        with open(path, encoding="utf-8") as f:
            return f.read()
    except (OSError, UnicodeDecodeError, EOFError):
        return Verdict("PARSE", "json", 0, -1)


def main(argv=None) -> int:
    argv = sys.argv[1:] if argv is None else argv
    if len(argv) != 1:
        print("Usage: python -m mortal_b200.validate_logs <DIR>", file=sys.stderr)
        return 2
    d = argv[0]
    paths = sorted(set(glob.glob(os.path.join(d, "**", "*.json"), recursive=True))
                   | set(glob.glob(os.path.join(d, "**", "*.json.gz"), recursive=True)))
    with ThreadPoolExecutor(min(32, os.cpu_count() or 1)) as pool:  # zlib and file reads release the GIL
        for lo in range(0, len(paths), CHUNK_LOGS):
            chunk = paths[lo:lo + CHUNK_LOGS]
            verdicts, enc = _validate(list(pool.map(_read, chunk)))
            for path, v, e in zip(chunk, verdicts, enc):
                if v is not None:
                    print(f"\nerror in log {path}\n{message(v, e)}", flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
