"""Helpers of the log-validation tests — TEST INFRASTRUCTURE: the emulated validator (emulv_validate_logs of
tests/host_emul/emul.cc, a single-lane host build of csrc/mjx_validate.cuh) and the oracle's restatement of bin/validate_logs.rs
(oracle/validate.cc, part of oracle/liboracle.so), over the same encoded logs."""
from __future__ import annotations

import ctypes as C
import json

import numpy as np

import emul_lib as E
import oracle_lib as O
from mortal_b200 import mjai_log
from mortal_b200.validate_logs import REASONS, STATUSES, EncodedLog, Verdict, encode_log, pack, to_verdict


def oracle_events(events):
    """mjai dicts -> the oracle's flat events; a hora's `has_deltas` carries the presence of `deltas` (bit 0) and of
    `ura_markers` (bit 1)"""
    arr = (O.OrcEvent * max(len(events), 1))()
    for i, ev in enumerate(events):
        arr[i] = O.event_from_json(ev)
        arr[i].has_deltas = int(ev.get("deltas") is not None) | int(ev.get("ura_markers") is not None) << 1
    return arr


def oracle_validate_events(arr, n):
    """the oracle's (status, reason, line, seat) codes of one log given as oracle_events()"""
    out = (C.c_int32 * 4)()
    L = O.lib()
    if L.orcv_validate_log(arr, n, out) != 0:
        raise RuntimeError(L.orcv_last_error().decode())
    return tuple(out)


def emul_run_packed(p) -> np.ndarray:
    """the emulated mjx_validate_logs over validate_logs.pack()'s arrays -> int32 [n, 4]"""
    n = len(p["ev_off"])
    out = np.zeros((n, 4), dtype=np.int32)
    rc = E.lib().emulv_validate_logs(n, p["hdr"].ctypes.data, p["ev_off"].ctypes.data, p["ev_cnt"].ctypes.data, len(p["hdr"]),
                                     p["kyoku"].ctypes.data, p["ky_off"].ctypes.data, len(p["kyoku"]), p["hora"].ctypes.data,
                                     p["hora_off"].ctypes.data, len(p["hora"]), out.ctypes.data)
    assert rc == 0
    return out


def emul_validate(texts):
    """validate_logs.validate_logs with the emulated kernel: [Verdict | None]"""
    enc = [encode_log(t) for t in texts]
    dev = [e for e in enc if isinstance(e, EncodedLog)]
    rows = emul_run_packed(pack(dev)) if dev else None
    out, k = [], 0
    for e in enc:
        if isinstance(e, Verdict):
            out.append(e)
        else:
            out.append(to_verdict(rows[k], e)); k += 1
    return out


def oracle_validate(text):
    """the oracle's verdict of one log text, with the same host-side parse step: Verdict | None"""
    e = encode_log(text)
    if isinstance(e, Verdict):
        return e
    events = [json.loads(t) for t in e.texts]
    return to_verdict(np.array(oracle_validate_events(oracle_events(events), len(events))), e)


def V(status, reason, line, seat=-1):
    assert status in STATUSES and reason in REASONS, (status, reason)
    return Verdict(status, reason, line, seat)


def emul_games(n, policy, seed0=123000, key=3):
    """`n` self-play games of the emulated environment under test policy `policy`, as mjai event lists"""
    nonces = np.arange(seed0, seed0 + n, dtype=np.uint64)
    keys = np.full(n, key, dtype=np.uint64)
    env = E.EmulEnv(nonces, keys, enable_quick_eval=(policy == 1))
    env.enable_log()
    acts = None
    for _ in range(100000):
        env.step(acts)
        acts = env.policy_test(policy)
        if env.num_live() == 0:
            break
    words, lens = env.read_log()
    env.close()
    return [[{"type": "start_game", "names": ["a", "b", "c", "d"], "seed": [int(nonces[t]), key]}]
            + mjai_log.decode_events(words[t, :int(lens[t])]) + [{"type": "end_game"}] for t in range(n)]
