"""libriichi bin/validate_logs.rs on the GPU: replay mjai logs through the four seats and report the first move a rule forbids.

    validate_logs(texts) -> [Verdict | None]      (None = the log is valid; all logs of a call run in one launch)
    python -m mortal_b200.validate_logs DIR       (every DIR/**/*.json and DIR/**/*.json.gz, in sorted order)

JSON decoding and the structural checks run on the host (dataset_codec.check_event, reported as PARSE); the rule checks and
the state updates run in the k_validate_logs kernel (csrc/mjx_validate.cuh). There is no CPU path: without a CUDA device
validate_logs raises.
"""
from __future__ import annotations

import glob
import gzip
import json
import os
import re
import sys
from dataclasses import dataclass

import numpy as np

from . import _lib
from .dataset_codec import HORA_WORDS, check_event, encode_events

STATUSES = ("OK", "CHECK", "UPDATE", "PARSE", "UNSUPPORTED")  # include/mjx.h mjx_verdict_status
CHUNK_LOGS = 4096  # logs decoded and validated per launch by the CLI: bounds its memory whatever the corpus size


def _read_reasons():
    """the reason names of include/mjx.h MJX_VALIDATE_REASONS, indexed by code (the header is their single definition)"""
    with open(os.path.join(os.path.dirname(_lib.HERE), "include", "mjx.h")) as f:
        text = f.read()
    block = text[text.index("#define MJX_VALIDATE_REASONS(X)"):]
    block = block[:block.index("#define MJX_REASON_ENUM_")]
    return tuple(name for _, name in re.findall(r'X\((\w+), "([^"]*)"\)', block))


REASONS = _read_reasons()


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


def _validate(texts, device: int = 0):
    _lib.init(device)  # no CUDA device: raises before any work, whatever the logs
    enc = [t if isinstance(t, Verdict) else encode_log(t) for t in texts]
    dev = [e for e in enc if isinstance(e, EncodedLog)]
    rows = run_packed(pack(dev), device) if dev else np.zeros((0, 4), dtype=np.int32)
    out, k = [], 0
    for e in enc:
        if isinstance(e, Verdict):
            out.append(e)
        else:
            out.append(to_verdict(rows[k], e)); k += 1
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
    for lo in range(0, len(paths), CHUNK_LOGS):
        chunk = paths[lo:lo + CHUNK_LOGS]
        verdicts, enc = _validate([_read(p) for p in chunk])
        for path, v, e in zip(chunk, verdicts, enc):
            if v is not None:
                print(f"\nerror in log {path}\n{message(v, e)}", flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
