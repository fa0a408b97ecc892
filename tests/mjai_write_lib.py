"""Helpers of the mjai writer tests — TEST INFRASTRUCTURE: the host build of csrc/mjx_mjai_write.cuh (tests/host_emul/
emul_mjai_write.cc), its bindings, and the comparison against CPython's float repr and the host writer (mortal_b200/mjai_log.py)."""
from __future__ import annotations

import ctypes as C

import numpy as np

import emul_lib as E


def emul_lib():
    """emul_lib.lib() with the emulated writer's entries declared"""
    L = E.lib()
    L.emulw_format_f32.restype = C.c_longlong
    L.emulw_format_f32.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong]
    L.emulw_render.restype = C.c_int
    L.emulw_render.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_longlong]
    L.emulw_meta_record.restype = C.c_int
    L.emulw_meta_record.argtypes = ([C.c_longlong] + [C.c_void_p] * 4 + [C.c_int, C.c_int] + [C.c_void_p] * 5 + [C.c_int, C.c_int]
                                    + [C.c_void_p] * 7 + [C.c_longlong, C.c_longlong])
    return L


def callback_lib():
    """emul_lib.pylib() with the formatter's comparison entries declared: they call back into this interpreter
    (PyOS_double_to_string) and need the GIL held"""
    L = E.pylib()
    L.emulw_sweep.restype = C.c_longlong
    L.emulw_sweep.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
    L.emulw_check.restype = C.c_longlong
    L.emulw_check.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
    return L


def format_f32(values) -> list[str]:
    """the emulated formatter over float32 values (or uint32 bit patterns)"""
    bits = np.ascontiguousarray(np.asarray(values).view(np.uint32) if np.asarray(values).dtype == np.float32 else values,
                                dtype=np.uint32)
    out = np.zeros(32 * len(bits) + 1, dtype=np.uint8)
    n = emul_lib().emulw_format_f32(bits.ctypes.data, len(bits), out.ctypes.data, out.size)
    assert n >= 0
    return out[:n].tobytes().decode("ascii").split("\n")[:-1]


def _py_fns():
    return C.cast(C.pythonapi.PyOS_double_to_string, C.c_void_p).value, C.cast(C.pythonapi.PyMem_Free, C.c_void_p).value


def sweep(lo: int, hi: int, step: int = 1):
    """(mismatches, first mismatching bit pattern) of the formatter against PyOS_double_to_string over [lo, hi)"""
    first = C.c_uint64(0)
    n = callback_lib().emulw_sweep(lo, hi, step, *_py_fns(), C.byref(first))
    return int(n), int(first.value)


def check(bits):
    """(mismatches, first mismatching bit pattern) of the formatter against PyOS_double_to_string over a list of patterns"""
    bits = np.ascontiguousarray(bits, dtype=np.uint32)
    first = C.c_uint64(0)
    n = callback_lib().emulw_check(bits.ctypes.data, len(bits), *_py_fns(), C.byref(first))
    return int(n), int(first.value)


def render(words, lens, bounds=None, recs=None):
    """the emulated count + fill over host arrays: (status int32 [n_games], list of text bytes per game (None: non-zero status))"""
    from mortal_b200 import mjai_write

    L = emul_lib()
    words = np.ascontiguousarray(words, dtype=np.uint64)
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    n, cap = words.shape
    a = mjai_write.render_args(bounds, recs)
    keep = [x for x in a.values() if isinstance(x, np.ndarray)]  # noqa: F841 — alive during the calls
    ptr = lambda x: x.ctypes.data if isinstance(x, np.ndarray) else None
    nbytes, status = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)
    args = (n, words.ctypes.data, lens.ctypes.data, cap, ptr(a["bounds"]), a["n_steps"], a["key_steps"], ptr(a["key"]), ptr(a["info"]),
            ptr(a["mask"]), ptr(a["q"]), ptr(a["i64"]), a["n_rec"])
    assert L.emulw_render(*args, nbytes.ctypes.data, status.ctypes.data, None, None, 0) == 0
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(nbytes, out=off[1:])
    out = np.zeros(max(int(off[-1]), 1), dtype=np.uint8)
    assert L.emulw_render(*args, nbytes.ctypes.data, status.ctypes.data, off.ctypes.data, out.ctypes.data, out.size) == 0
    return status, [out[off[g]:off[g + 1]].tobytes() if status[g] == 0 else None for g in range(n)]


class EmulRecords:
    """DeviceMetaRecorder's record arrays on the host, appended by the host build of k_meta_record (emulw_meta_record)"""

    def __init__(self, cap):
        self.L = emul_lib()
        self.cap, self.count, self.calls, self.max_cycle = cap, 0, [], -1
        self.table, self.cycle = np.zeros(cap, np.int32), np.zeros(cap, np.int32)
        self.seat, self.info = np.zeros(cap, np.uint8), np.zeros((cap, 4), np.int32)
        self.mask, self.q, self.call = np.zeros(cap, np.uint64), np.zeros((cap, 46), np.float32), np.zeros(cap, np.int32)

    def record(self, cycle, q, row_table, row_seat, actions, masks, *, idx=None, greedy=None, call_ids=None, call=0, obs=None,
               row_cap=None, n=None):
        c = lambda x, dt: None if x is None else np.ascontiguousarray(x, dtype=dt)
        q, idx, greedy, call_ids = c(q, np.float32), c(idx, np.int64), c(greedy, np.uint8), c(call_ids, np.int32)
        row_table, row_seat, actions = c(row_table, np.int32), c(row_seat, np.uint8), c(actions, np.int64)
        masks, obs = c(masks, np.uint8), c(obs, np.float32)
        n = len(q) if n is None else n
        ptr = lambda x: None if x is None else x.ctypes.data
        rc = self.L.emulw_meta_record(n, ptr(idx), ptr(q), ptr(greedy), ptr(call_ids), call, cycle, ptr(row_table), ptr(row_seat),
                                      ptr(actions), ptr(masks), ptr(obs), 0 if obs is None else obs.shape[1],
                                      len(actions) if row_cap is None else row_cap, self.table.ctypes.data, self.cycle.ctypes.data,
                                      self.seat.ctypes.data, self.info.ctypes.data, self.mask.ctypes.data, self.q.ctypes.data,
                                      self.call.ctypes.data, self.count, self.cap)
        assert rc == 0
        self.count = min(self.count + n, self.cap)
        self.max_cycle = max(self.max_cycle, cycle)

    def render_recs(self):
        """the recorder_records form of these records (what DeviceMetaRecorder.device_args sorts on the device)"""
        n = self.count
        calls = np.array(self.calls or [(0, 0)], dtype=np.int64).reshape(-1, 2)
        call = self.call[:n].astype(np.int64)
        i64 = np.where((call >= 0)[:, None], calls[np.clip(call, 0, None)], 0)
        return dict(table=self.table[:n].astype(np.int64), cycle=self.cycle[:n].astype(np.int64), seat=(self.seat[:n] & 3).astype(np.int64),
                    kan=((self.seat[:n] >> 2) & 1).astype(np.int64), action=self.info[:n, 0].astype(np.int64), flags=self.info[:n, 1],
                    shanten=self.info[:n, 2].astype(np.int64), row=self.info[:n, 3].astype(np.int64), mask=self.mask[:n], q=self.q[:n],
                    i64=i64)
