"""Helpers of the single-viewpoint loader tests — TEST INFRASTRUCTURE: the log the mjai protocol shows one seat, the scan
k_replay_viewpoints makes restated over mjai events, and the host build of the replay with that scan (tests/host_emul/emul_viewpoint.cc:
emul.cc plus the scan entry) behind EmulViewReplay, the emulated stand-in for ReplayEnv with viewpoints()."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import emul_lib as E

EMUL_SRC = os.path.join(E.ROOT, "tests", "host_emul", "emul_viewpoint.cc")
EMUL_SO = os.path.join(E.ROOT, "tests", "host_emul", "libmjx_emul_viewpoint.so")
_emul = None


def build_emul(so=EMUL_SO, extra=()):
    deps = [EMUL_SRC, E.SRC] + [os.path.join(E.CSRC, f) for f in os.listdir(E.CSRC) if f.endswith((".cuh", ".h"))]
    if extra or not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O2" if not extra else "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-DMJX_HOST_EMUL",
                               "-ffp-contract=off", "-I" + E.CSRC, "-Wno-unknown-pragmas", *extra, "-o", so, EMUL_SRC])
    return so


def build():
    build_emul()


def emul_lib(path=None):
    """the host build with the scan entry, bound like emul_lib.lib() binds emul.cc's; `path` loads another build (the sanitizer
    run's)"""
    global _emul
    if _emul is None or path is not None:
        saved = E._lib, E.build
        try:  # emul_lib.lib() binds and initialises whatever its build() returns; its own library is left as it was
            E._lib, E.build = None, (lambda: path or build_emul())
            L = E.lib()
        finally:
            E._lib, E.build = saved
        L.emul_replay_viewpoints.argtypes = [C.c_void_p, C.c_void_p]
        _emul = L
    return _emul


class EmulViewReplay(E.EmulReplay):
    """emul_lib.EmulReplay on the library with the scan: viewpoints() is mjx_env_replay_viewpoints / ReplayEnv.viewpoints()"""

    def __init__(self, jobs, always_include_kan_select=True):
        self.L = emul_lib()
        self.jobs = {k: np.ascontiguousarray(v) for k, v in jobs.items()}
        j = self.jobs
        self.n_tables = len(j["players"])
        self.row_cap = self.n_tables * 3
        self._h = self.L.emul_replay_create(self.n_tables, j["hdr"].ctypes.data, j["ev_off"].ctypes.data, j["ev_cnt"].ctypes.data,
                                            len(j["hdr"]), j["kyoku"].ctypes.data, j["ky_off"].ctypes.data, len(j["kyoku"]),
                                            j["players"].ctypes.data, int(always_include_kan_select))
        self.live = self.n_tables

    def viewpoints(self):
        """single-viewpoint logs replay from the player's own seat; returns the scan result per job (-1 = not marked, else the
        mask of hidden seats)"""
        m = np.zeros(self.n_tables, dtype=np.int32)
        self.L.emul_replay_viewpoints(self._h, m.ctypes.data)
        return m


def named(events):
    """the log with four distinct player names (`<name>.<seat>`), so that player_names selects exactly one seat"""
    first = dict(events[0])
    names = list(first.get("names", ["", "", "", ""]))
    first["names"] = [f"{nm}.{s}" for s, nm in enumerate(names)]
    return [first] + list(events[1:])


def viewpoint(events, p):
    """the log as seat p's mjai client receives it: the other seats' haipai are 13 x "?" and their draws "pai": "?"; with
    named()'s distinct names"""
    out = []
    for ev in named(events):
        if ev["type"] == "start_kyoku":
            ev = {**ev, "tehais": [list(h) if s == p else ["?"] * 13 for s, h in enumerate(ev["tehais"])]}
        elif ev["type"] == "tsumo" and ev["actor"] != p:
            ev = {**ev, "pai": "?"}
        out.append(ev)
    return out


def hidden_seats(events):
    """the mask k_replay_viewpoints computes: bit s when a haipai tile of seat s or a tsumo of seat s is "?" """
    m = 0
    for ev in events:
        if ev["type"] == "start_kyoku":
            for s, h in enumerate(ev["tehais"]):
                if "?" in h:
                    m |= 1 << s
        elif ev["type"] == "tsumo" and ev["pai"] == "?":
            m |= 1 << ev["actor"]
    return m
