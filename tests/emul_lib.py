"""Builds and binds tests/host_emul/libmjx_emul.so — TEST INFRASTRUCTURE: every tests/host_emul/*.cc (single-lane host builds
of the product's device sources, -DMJX_HOST_EMUL) linked into one library, with every entry of their extern "C" blocks bound
from its C definition. Never used by mortal_b200/."""
import ctypes as C
import glob
import os
import subprocess
import tempfile

import numpy as np

from mortal_b200 import _cdecl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST_EMUL = os.path.join(ROOT, "tests", "host_emul")
SO = os.path.join(HOST_EMUL, "libmjx_emul.so")
ASAN_SO = os.path.join(HOST_EMUL, "libmjx_emul_asan.so")
CSRC = os.path.join(ROOT, "mortal_b200", "csrc")
DATA_DIR = os.path.join(ROOT, "mortal_b200", "data")
FLAGS = ["-g", "-std=c++17", "-fPIC", "-DMJX_HOST_EMUL", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-I" + CSRC]
_lib = _pylib = None


def build(sanitize=False):
    """Compiles the library when it is older than a source, a csrc/ file, include/mjx.h or this file (the flags); returns its
    path. sanitize=True builds the same sources under ASan + UBSan into a file of its own, so it never replaces the normal build."""
    so = ASAN_SO if sanitize else SO
    srcs = sorted(glob.glob(os.path.join(HOST_EMUL, "*.cc")))
    deps = srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "mjx.h"), __file__]
    if os.path.exists(so) and all(os.path.getmtime(d) <= os.path.getmtime(so) for d in deps):
        return so
    opt = ["-O1", "-fsanitize=address,undefined", "-fno-omit-frame-pointer"] if sanitize else ["-O2"]
    with tempfile.TemporaryDirectory() as tmp:  # one compiler per source, in parallel: emul.cc alone takes ~10 s
        objs = [os.path.join(tmp, os.path.basename(s) + ".o") for s in srcs]
        procs = [subprocess.Popen(["g++", *opt, *FLAGS, "-c", "-o", o, s]) for s, o in zip(srcs, objs)]
        if [p.wait() for p in procs] != [0] * len(procs):
            raise RuntimeError("compiling tests/host_emul failed")
        subprocess.check_call(["g++", *opt, "-shared", "-Wl,--no-undefined", "-o", so, *objs])
    return so


def _entries():
    """the ctypes signatures of every extern "C" function of tests/host_emul/*.cc"""
    srcs = sorted(glob.glob(os.path.join(HOST_EMUL, "*.cc")))
    return _cdecl.functions("".join(open(s).read() for s in srcs), "emul")


def lib(sanitize=False):
    """The library, loaded once, with every entry bound and the lookup tables loaded. A sanitizer run calls lib(sanitize=True)
    before anything else loads the library."""
    global _lib
    if _lib is None:
        L = _cdecl.bind(C.CDLL(build(sanitize)), _entries())
        if L.emul_init(DATA_DIR.encode()) != 0:
            raise RuntimeError(L.emul_last_error().decode())
        _lib = L
    elif sanitize and _lib._name != ASAN_SO:
        raise RuntimeError("libmjx_emul.so is already loaded without sanitizers")
    return _lib


def pylib():
    """lib()'s file loaded again with ctypes.PyDLL, whose calls hold the GIL: for entries that call back into Python"""
    global _pylib
    if _pylib is None:
        _pylib = _cdecl.bind(C.PyDLL(lib()._name), _entries())
    return _pylib


def run(nonces, keys, *, shuffle_kind=0, quick_eval=True, policy_kind=1, trace_cap=0, max_cycles=0, agari_guard=False):
    n = len(nonces)
    nonces = np.ascontiguousarray(nonces, dtype=np.uint64)
    keys = np.ascontiguousarray(keys, dtype=np.uint64)
    scores = np.zeros((n, 4), dtype=np.int32)
    ranks = np.zeros((n, 4), dtype=np.uint8)
    steps = np.zeros(n, dtype=np.int32)
    errs = np.zeros(n, dtype=np.int32)
    trace = np.zeros((max(trace_cap, 1), 6), dtype=np.int64)
    tl = C.c_int64(0)
    rc = lib().emul_run(n, nonces.ctypes.data, keys.ctypes.data, shuffle_kind, int(quick_eval), policy_kind,
                        scores.ctypes.data, ranks.ctypes.data, steps.ctypes.data, errs.ctypes.data,
                        trace.ctypes.data if trace_cap else None, trace_cap, C.byref(tl), max_cycles, int(agari_guard))
    assert rc == 0
    out = dict(scores=scores, ranks=ranks, steps=steps, errs=errs, n_rows=tl.value)
    if trace_cap:
        assert tl.value <= trace_cap
        out["trace"] = trace[: tl.value]
    return out


class EmulEnv:
    """Host-emulated stand-in with the stepping surface of mortal_b200.BatchEnv (numpy instead of torch)."""

    def __init__(self, nonces, keys, *, shuffle_kind=0, enable_quick_eval=True):
        self.L = lib()
        nonces = np.ascontiguousarray(nonces, dtype=np.uint64)
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        self.n_tables = len(nonces)
        self.row_cap = self.n_tables * 3
        self._h = self.L.emul_env_create(self.n_tables, nonces.ctypes.data, keys.ctypes.data, shuffle_kind,
                                         int(enable_quick_eval))
        self.live = self.n_tables

    def close(self):
        if self._h:
            self.L.emul_env_destroy(self._h)
            self._h = None

    def step(self, actions=None):
        a = None if actions is None else np.ascontiguousarray(actions, dtype=np.int64)
        self.live = self.L.emul_env_step(self._h, None if a is None else a.ctypes.data)

    def num_rows(self):
        return self.L.emul_env_num_rows(self._h)

    def num_live(self):
        return self.live

    def rows(self):
        n = self.num_rows()
        rt = np.zeros(n, dtype=np.int32); rs = np.zeros(n, dtype=np.uint8); m = np.zeros((n, 46), dtype=np.uint8)
        self.L.emul_env_rows(self._h, rt.ctypes.data, rs.ctypes.data, m.ctypes.data)
        return rt, rs, m.astype(bool)

    def policy_test(self, kind):
        a = np.full(self.row_cap, 45, dtype=np.int64)
        self.L.emul_env_policy_test(self._h, kind, a.ctypes.data)
        return a

    def enable_grp(self, cap=32):
        self._grp_cap = cap
        self.L.emul_env_enable_grp(self._h, cap)

    def read_grp(self):
        feat = np.zeros((self.n_tables, self._grp_cap, 7), dtype=np.int32); cnt = np.zeros(self.n_tables, dtype=np.int32)
        self.L.emul_env_read_grp(self._h, feat.ctypes.data, cnt.ctypes.data)
        out = []
        for t in range(self.n_tables):
            f = feat[t, : cnt[t]].astype(np.float64)
            f[:, 3:] /= 10000.0
            out.append(f)
        return out

    def enable_log(self, cap=8192):
        self._log_cap = cap
        self.L.emul_env_enable_log(self._h, cap)

    def log_lens(self):
        lens = np.zeros(self.n_tables, dtype=np.int32)
        self.L.emul_env_log_lens(self._h, lens.ctypes.data)
        return lens

    def read_log(self):
        words = np.zeros((self.n_tables, self._log_cap), dtype=np.uint64)
        lens = np.zeros(self.n_tables, dtype=np.int32)
        self.L.emul_env_read_log(self._h, words.ctypes.data, lens.ctypes.data)
        assert (lens <= self._log_cap).all()
        return words, lens

    def encode_invisible(self, version=4):
        rows = 211 if version == 1 else 217
        out = np.zeros((self.num_rows(), rows, 34), dtype=np.float32)
        self.L.emul_env_encode_invisible(self._h, out.ctypes.data, version)
        return out

    def encode_obs(self, sp=False, version=4):
        rows = {1: 938, 2: 942, 3: 934, 4: 1012}[version]
        obs = np.zeros((self.num_rows(), rows, 34), dtype=np.float32)
        self.L.emul_env_encode_obs_v(self._h, obs.ctypes.data, int(sp), version)
        return obs


class EmulReplay(EmulEnv):
    """Host-emulated stand-in for the replay mode of mortal_b200.BatchEnv (mjx_env_create_replay / mjx_env_replay_step)."""

    def __init__(self, jobs, always_include_kan_select=True):
        self.L = lib()
        self.jobs = {k: np.ascontiguousarray(v) for k, v in jobs.items()}
        j = self.jobs
        self.n_tables = len(j["players"])
        self.row_cap = self.n_tables * 3
        self._h = self.L.emul_replay_create(self.n_tables, j["hdr"].ctypes.data, j["ev_off"].ctypes.data, j["ev_cnt"].ctypes.data,
                                            len(j["hdr"]), j["kyoku"].ctypes.data, j["ky_off"].ctypes.data, len(j["kyoku"]),
                                            j["players"].ctypes.data, int(always_include_kan_select))
        self.live = self.n_tables

    def replay_step(self):
        self.live = self.L.emul_replay_step(self._h)

    def trust_seeds(self, nonces, keys, shuffle_kind=0):
        n_ = np.ascontiguousarray(nonces, dtype=np.uint64); k_ = np.ascontiguousarray(keys, dtype=np.uint64)
        self.L.emul_replay_trust_seeds(self._h, n_.ctypes.data, k_.ctypes.data, shuffle_kind)

    def encode_invisible(self, version=4):
        out = np.zeros((self.num_rows(), 211 if version == 1 else 217, 34), dtype=np.float32)
        self.L.emul_replay_encode_invisible(self._h, out.ctypes.data, version)
        return out

    def viewpoints(self):
        """mjx_env_replay_viewpoints / ReplayEnv.viewpoints(): single-viewpoint logs replay from the player's own seat; returns
        the scan result per job (-1 = not marked, else the mask of hidden seats)"""
        m = np.zeros(self.n_tables, dtype=np.int32)
        self.L.emul_replay_viewpoints(self._h, m.ctypes.data)
        return m

    def row_labels(self):
        n = self.num_rows()
        lab = np.zeros(max(n, 1), dtype=np.int64); meta = np.zeros((max(n, 1), 4), dtype=np.uint8)
        self.L.emul_replay_rows(self._h, lab.ctypes.data, meta.ctypes.data)
        return lab[:n], meta[:n]

    def errs(self):
        e = np.zeros(self.n_tables, dtype=np.int32)
        self.L.emul_env_errs(self._h, e.ctypes.data)
        return e
