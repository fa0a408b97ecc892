"""Helpers of the statistics tests — TEST INFRASTRUCTURE: the host build of csrc/mjx_stat.cuh (tests/host_emul/emul_stat.cc),
a host encoder of the arrays k_stat_logs reads (event words and payloads from dataset_codec.encode_events, the per-event deltas
from the json events), and the host path's per-log expectation."""
from __future__ import annotations

import ctypes as C

import numpy as np

import emul_lib as E
from mortal_b200 import dataset_codec
from mortal_b200.stat import Stat, _read_counters

NAMES = _read_counters()  # include/mjx.h MJX_STAT_COUNTERS
STATUS = {0: "ok", 1: "not start_game", 2: "no deltas", 3: "capacity"}  # include/mjx.h mjx_stat_status


def emul_lib():
    """emul_lib.lib() with the emulated kernel's entries declared"""
    L = E.lib()
    L.emuls_stat_logs.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_longlong,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.emuls_line_deltas.argtypes = [C.c_char_p, C.c_longlong, C.c_void_p]
    return L


def encode_deltas(events):
    """the deltas arrays of mjx_mjai_fill_deltas_dev for one log: int32 [n, 4] (zero where not written) and uint8 [n]"""
    d = np.zeros((len(events), 4), dtype=np.int32)
    has = np.zeros(len(events), dtype=np.uint8)
    for k, ev in enumerate(events):
        if ev["type"] in ("hora", "ryukyoku") and ev.get("deltas") is not None:
            d[k] = ev["deltas"]
            has[k] = 1
    return d, has


def encode(games):
    """event lists -> the arrays k_stat_logs reads, in the layout of the decoder's (concatenated, per-log offsets)"""
    hdr, ky, dl, hs = [], [], [], []
    n = len(games)
    ev_off, ev_cnt, ky_off = (np.zeros(n, dtype=np.int32) for _ in range(3))
    ne = nk = 0
    for i, events in enumerate(games):
        h, p = dataset_codec.encode_events(events)
        d, has = encode_deltas(events)
        ev_off[i], ev_cnt[i], ky_off[i] = ne, len(h), nk
        ne += len(h); nk += len(p)
        hdr.append(np.asarray(h, dtype=np.uint64)); ky.append(np.asarray(p, dtype=np.uint64).reshape(-1)); dl.append(d); hs.append(has)
    cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs) if xs else np.zeros(0, dtype=dt), dtype=dt)
    return dict(hdr=cat(hdr, np.uint64), ev_off=ev_off, ev_cnt=ev_cnt, kyoku=cat(ky, np.uint64), ky_off=ky_off,
                deltas=np.ascontiguousarray(np.concatenate(dl) if dl else np.zeros((0, 4)), dtype=np.int32), has=cat(hs, np.uint8))


def run_emul(a, seats, n_hdr=None, n_kyoku_words=None):
    """the emulated kernel over encode()'s arrays -> (int64 [n, MJX_STAT_N], int32 [n]); n_hdr / n_kyoku_words override the
    capacities (hostile-array tests)"""
    L = emul_lib()
    n = len(a["ev_off"])
    seats = np.ascontiguousarray(seats, dtype=np.uint8)
    out = np.full((n, len(NAMES)), -1, dtype=np.int64)
    status = np.full(n, -1, dtype=np.int32)
    ptr = lambda x: x.ctypes.data if x.size else None
    rc = L.emuls_stat_logs(n, ptr(a["hdr"]), a["ev_off"].ctypes.data, a["ev_cnt"].ctypes.data,
                           len(a["hdr"]) if n_hdr is None else n_hdr, ptr(a["kyoku"]), a["ky_off"].ctypes.data,
                           len(a["kyoku"]) if n_kyoku_words is None else n_kyoku_words, ptr(a["deltas"]), ptr(a["has"]),
                           seats.ctypes.data, out.ctypes.data, status.ctypes.data)
    assert rc == 0
    return out, status


def line_deltas(line: bytes):
    """mjai_line_deltas of the decoder (host build) -> (has_deltas, [4 ints])"""
    d = np.zeros(4, dtype=np.int32)
    has = emul_lib().emuls_line_deltas(line, len(line), d.ctypes.data)
    return bool(has), [int(x) for x in d]


def host_row(events, mask):
    """the sum of Stat.from_game over the seats of `mask`, as a counter row in MJX_STAT_COUNTERS order, or None where Python
    raises (which must be a non-zero status on the device)"""
    st = Stat()
    try:
        for s in range(4):
            if mask >> s & 1:
                st = st + Stat.from_game(events, s)
    except Exception:  # noqa: BLE001
        return None
    return np.array([getattr(st, c) for c in NAMES], dtype=np.int64)


def seat_mask(events, name):
    return sum(1 << i for i, n in enumerate(events[0].get("names", [])) if n == name and i < 4)
