"""Helpers of the observation codec tests — TEST INFRASTRUCTURE: the host build of csrc/mjx_obs_pack.cuh
(tests/host_emul/emul_obs_pack.cc) and observation fixtures of every version from the oracle."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import emul_lib as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROWS = {(1, False): 938, (2, False): 942, (3, False): 934, (4, False): 1012, (1, True): 211, (2, True): 217, (3, True): 217,
        (4, True): 217}


def emul_lib():
    """emul_lib.lib() with the emulated codec's entries declared"""
    L = E.lib()
    L.emulp_record_bytes.restype = C.c_int
    L.emulp_record_bytes.argtypes = [C.c_int, C.c_int]
    L.emulp_pack.restype = C.c_int
    L.emulp_pack.argtypes = [C.c_int, C.c_int, C.c_longlong, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p]
    L.emulp_unpack.restype = C.c_int
    L.emulp_unpack.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_void_p]
    L.emulp_value_rows.restype = C.c_int
    L.emulp_value_rows.argtypes = [C.c_int, C.c_int, C.c_void_p]
    return L


def record_bytes(version, invisible):
    return emul_lib().emulp_record_bytes(version, int(invisible))


def value_rows(version, invisible):
    buf = np.zeros(96, dtype=np.int16)
    n = emul_lib().emulp_value_rows(version, int(invisible), buf.ctypes.data)
    assert n >= 0
    return buf[:n].astype(np.int64)


def pack(x, version, invisible, pitch=None, n=None):
    """emulp_pack over float32 [n, rows, 34] (or a flat buffer with `pitch` floats between samples) -> (rc, records uint8
    [n, record_bytes], status int32 [n])"""
    x = np.ascontiguousarray(x, dtype=np.float32)
    n = len(x) if n is None else n
    pitch = ROWS.get((version, bool(invisible)), 938) * 34 if pitch is None else pitch
    rb = max(record_bytes(version, invisible), 0)
    rec = np.full((max(n, 0), rb), 0xA5, dtype=np.uint8)
    status = np.full(max(n, 0), -7, dtype=np.int32)
    rc = emul_lib().emulp_pack(version, int(invisible), n, x.ctypes.data if x.size else None, pitch, rec.ctypes.data if rec.size else None,
                               status.ctypes.data if n > 0 else None)
    return rc, rec, status


def unpack(rec, idx, version, invisible, n_records=None):
    """emulp_unpack -> (rc, float32 [len(idx), rows, 34])"""
    rec = np.ascontiguousarray(rec, dtype=np.uint8)
    idx = np.ascontiguousarray(idx, dtype=np.int64)
    out = np.full((len(idx), ROWS.get((version, bool(invisible)), 938), 34), np.nan, dtype=np.float32)
    rc = emul_lib().emulp_unpack(version, int(invisible), rec.ctypes.data if rec.size else None, len(rec) if n_records is None else n_records,
                                 idx.ctypes.data if idx.size else None, len(idx), out.ctypes.data if out.size else None)
    return rc, out


def golden_events():
    import json

    with open(os.path.join(ROOT, "tests", "golden", "golden_game.jsonl")) as f:
        return [{k: v for k, v in json.loads(ln).items() if k != "meta"} for ln in f if ln.strip()]


def sample_obs(version, seed=5, n_tables=8, steps=60):
    """observations of self-play decisions from oracle_lib.run_sample_obs (invisible=True) -> (obs, invisible), with kan-select
    rows asked for at every sampled step"""
    import oracle_lib as O

    rng = np.random.default_rng(seed)
    nonces = np.repeat(np.arange(4000 + seed * 100, 4000 + seed * 100 + n_tables // 4, dtype=np.uint64), 4)
    keys = np.full(n_tables, 0x3000 + seed, dtype=np.uint64)
    samples = np.array([(t, s, seat, ks) for t in range(n_tables) for s in rng.choice(steps, 12, replace=False) for seat in range(4)
                        for ks in (0, 1)], dtype=np.int64)
    obs, _, found, inv = O.run_sample_obs(nonces, keys, samples, version=version, max_steps=steps + 2, invisible=True)
    return obs[found], inv[found]
