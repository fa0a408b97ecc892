"""Device-resident batch environment: Python handle over mjx_env (include/mjx.h).

Mirrors the loop of libriichi's BatchGame::run (arena/game.rs:230-316): `step()` = one iteration
for every live table (commit the previous decisions, poll to the next decision point), the rows it
emits are what MortalBatchAgent would hand to `engine.react_batch` (agent/mortal.rs:114-159).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib


class _CudaView:
    """Zero-copy torch view of a device buffer owned by the C library (__cuda_array_interface__ v2)."""

    def __init__(self, ptr: int, shape, typestr: str):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False),
                                         "version": 2, "strides": None}


class BatchEnv:
    def __init__(self, nonces, keys, *, obs_version: int = 4, shuffle_kind: int = 0, enable_quick_eval: bool = True,
                 device: int = 0):
        import torch

        if not torch.cuda.is_available():
            raise _lib.MjxError("mortal_b200.BatchEnv needs a CUDA device (there is no CPU fallback)")
        self.torch = torch
        self.device = torch.device("cuda", device)
        torch.cuda.set_device(self.device)
        _lib.init(device)
        self.L = _lib.load()
        nonces = np.ascontiguousarray(nonces, dtype=np.uint64)
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        assert nonces.shape == keys.shape and nonces.ndim == 1
        self.n_tables = int(nonces.shape[0])
        self.obs_version = obs_version
        self.obs_rows = self.L.mjx_obs_rows(obs_version)
        h = C.c_void_p()
        _lib.check(self.L.mjx_env_create(C.byref(h), self.n_tables, nonces.ctypes.data, keys.ctypes.data, obs_version,
                                         shuffle_kind, int(enable_quick_eval)), "mjx_env_create")
        self._h = h
        self._bind_views()

    def _bind_views(self):
        torch, h = self.torch, self._h
        self.row_cap = self.L.mjx_env_row_cap(h)
        as_t = lambda ptr, shape, ts: torch.as_tensor(_CudaView(ptr, shape, ts), device=self.device)
        self._as_t = as_t
        self.masks = as_t(self.L.mjx_env_masks(h), (self.row_cap, 46), "|u1").view(torch.bool)
        self.row_table = as_t(self.L.mjx_env_row_table(h), (self.row_cap,), "<i4")
        self.row_seat = as_t(self.L.mjx_env_row_seat(h), (self.row_cap,), "|u1")
        self.row_step = as_t(self.L.mjx_env_row_step(h), (self.row_cap,), "<u4")
        self.n_rows_dev = as_t(self.L.mjx_env_num_rows_dev(h), (1,), "<i4")
        self._obs = None

    def close(self):
        if getattr(self, "_h", None):
            self.L.mjx_env_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return C.c_void_p(self.torch.cuda.current_stream(self.device).cuda_stream)

    def step(self, actions=None, q_values=None) -> None:
        """actions: int64 cuda tensor [row_cap] indexed by the previous step's rows (None on the first step);
        q_values: float32 cuda tensor [row_cap, 46], only needed when an agari guard is set."""
        ptr = qptr = None
        if actions is not None:
            assert actions.dtype == self.torch.int64 and actions.is_cuda and actions.is_contiguous()
            assert actions.numel() >= self.row_cap
            ptr = C.c_void_p(actions.data_ptr())
        if q_values is not None:
            assert q_values.dtype == self.torch.float32 and q_values.is_cuda and q_values.is_contiguous()
            assert q_values.shape == (self.row_cap, 46)
            qptr = C.c_void_p(q_values.data_ptr())
        _lib.check(self.L.mjx_env_step(self._h, ptr, qptr, self._stream()), "mjx_env_step")

    def set_agari_guard(self, flags) -> None:
        """flags: None or uint8 array [n_tables, 4] (1 = that seat's engine has enable_rule_based_agari_guard)."""
        if flags is None:
            _lib.check(self.L.mjx_env_set_agari_guard(self._h, None), "mjx_env_set_agari_guard")
            return
        f = np.ascontiguousarray(flags, dtype=np.uint8)
        assert f.shape == (self.n_tables, 4)
        _lib.check(self.L.mjx_env_set_agari_guard(self._h, f.ctypes.data), "mjx_env_set_agari_guard")

    def set_quick_eval(self, flags) -> None:
        """flags: None or uint8 array [n_tables, 4] (1 = that seat's engine has enable_quick_eval)."""
        if flags is None:
            _lib.check(self.L.mjx_env_set_quick_eval(self._h, None), "mjx_env_set_quick_eval")
            return
        f = np.ascontiguousarray(flags, dtype=np.uint8)
        assert f.shape == (self.n_tables, 4)
        _lib.check(self.L.mjx_env_set_quick_eval(self._h, f.ctypes.data), "mjx_env_set_quick_eval")

    def set_obs_version(self, version: int) -> None:
        """switch the version encode_obs / encode_obs_host produce (agent/mortal.rs:54-74: every agent has its own)"""
        _lib.check(self.L.mjx_env_set_obs_version(self._h, int(version)), "mjx_env_set_obs_version")
        if version != self.obs_version:
            self.obs_version = int(version)
            self.obs_rows = self.L.mjx_obs_rows(version)
            self._obs = None

    def obs_buffer(self):
        if self._obs is None:
            self._obs = self.torch.empty((self.row_cap, self.obs_rows, 34), dtype=self.torch.float32, device=self.device)
        return self._obs

    def encode_obs(self, out=None):
        """Encode the current rows; returns the [row_cap, C, 34] buffer (first num_rows() rows valid)."""
        out = self.obs_buffer() if out is None else out
        assert out.dtype == self.torch.float32 and out.is_contiguous() and out.shape[1:] == (self.obs_rows, 34)
        assert out.shape[0] >= self.row_cap
        _lib.check(self.L.mjx_env_encode_obs(self._h, C.c_void_p(out.data_ptr()), self._stream()), "mjx_env_encode_obs")
        return out

    def encode_obs_host(self, obs_host, masks_host) -> int:
        """Encode the current rows into HOST tensors (pinned for speed): obs_host f32 [>=row_cap, C, 34], masks_host
        bool/uint8 [>=row_cap, 46]. The D2H copy of rows 0..888 overlaps the single-player kernels. Returns num_rows."""
        assert obs_host.dtype == self.torch.float32 and obs_host.is_contiguous() and not obs_host.is_cuda
        assert obs_host.shape[0] >= self.row_cap and tuple(obs_host.shape[1:]) == (self.obs_rows, 34)
        assert masks_host.element_size() == 1 and masks_host.is_contiguous() and not masks_host.is_cuda
        assert masks_host.shape[0] >= self.row_cap and masks_host.shape[1] == 46
        n = C.c_int(0)
        _lib.check(self.L.mjx_env_encode_obs_host(self._h, C.c_void_p(self.obs_buffer().data_ptr()), C.c_void_p(obs_host.data_ptr()),
                                                  C.c_void_p(masks_host.data_ptr()), C.byref(n), self._stream()),
                   "mjx_env_encode_obs_host")
        return n.value

    def encode_invisible(self, version: int = None):
        """Invisible (oracle) observation of the current rows (board.rs:680-782): [row_cap, 211 | 217, 34] f32 on the device."""
        version = self.obs_version if version is None else version
        rows = self.L.mjx_oracle_obs_rows(version)
        if getattr(self, "_inv", None) is None or self._inv.shape[1] != rows:
            self._inv = self.torch.empty((self.row_cap, rows, 34), dtype=self.torch.float32, device=self.device)
        _lib.check(self.L.mjx_env_encode_invisible(self._h, C.c_void_p(self._inv.data_ptr()), version, self._stream()),
                   "mjx_env_encode_invisible")
        return self._inv

    def encode_obs_host_begin(self, obs_host, masks_host) -> int:
        """Asynchronous half of encode_obs_host: enqueue encode + D2H and return num_rows as soon as it is known."""
        assert obs_host.dtype == self.torch.float32 and obs_host.is_contiguous() and not obs_host.is_cuda
        assert obs_host.shape[0] >= self.row_cap and tuple(obs_host.shape[1:]) == (self.obs_rows, 34)
        assert masks_host.element_size() == 1 and masks_host.is_contiguous() and not masks_host.is_cuda
        n = C.c_int(0)
        _lib.check(self.L.mjx_env_encode_obs_host_begin(self._h, C.c_void_p(self.obs_buffer().data_ptr()), C.c_void_p(obs_host.data_ptr()),
                                                        C.c_void_p(masks_host.data_ptr()), C.byref(n), self._stream()),
                   "mjx_env_encode_obs_host_begin")
        return n.value

    def encode_obs_host_finish(self) -> None:
        _lib.check(self.L.mjx_env_encode_obs_host_finish(self._h), "mjx_env_encode_obs_host_finish")

    def set_sp(self, enable: bool) -> None:
        _lib.check(self.L.mjx_env_set_sp(self._h, int(enable)), "mjx_env_set_sp")

    def sp_overflows(self) -> int:
        n = C.c_int(0)
        _lib.check(self.L.mjx_env_sp_overflows(self._h, self._stream(), C.byref(n)), "mjx_env_sp_overflows")
        return n.value

    def sp_stats(self):
        """(states, edges, [states per level slot D3 W3 D2 W2 D1 W1 D0 W0]) of the last step's single-player DP"""
        out = (C.c_int * 10)()
        _lib.check(self.L.mjx_env_sp_stats(self._h, self._stream(), out), "mjx_env_sp_stats")
        return out[0], out[1], list(out[2:10])

    def enable_log(self, words_per_table: int = 8192) -> None:
        """Record every table's mjai events on device (arena/result.rs GameResult.game_log); call before the first step."""
        _lib.check(self.L.mjx_env_enable_log(self._h, int(words_per_table)), "mjx_env_enable_log")
        self._log_cap = int(words_per_table)
        self.log_len = self._as_t(self.L.mjx_env_log_len_dev(self._h), (self.n_tables,), "<i4")  # words written so far, per table
        self.log_words = self._as_t(self.L.mjx_env_log_words_dev(self._h), (self.n_tables, self._log_cap), "<i8")  # the words (bits)

    def read_log(self):
        """-> (words uint64 [n_tables, cap], lengths int32 [n_tables]); decode with mortal_b200.mjai_log"""
        words = np.zeros((self.n_tables, self._log_cap), dtype=np.uint64)
        lens = np.zeros(self.n_tables, dtype=np.int32)
        _lib.check(self.L.mjx_env_read_log(self._h, self._stream(), words.ctypes.data, lens.ctypes.data), "mjx_env_read_log")
        if (lens > self._log_cap).any():
            raise RuntimeError(f"event log overflow: {int(lens.max())} words > capacity {self._log_cap}")
        return words, lens

    def enable_grp(self, max_kyoku: int = 32) -> None:
        """Record the GRP feature row of every kyoku on device (dataset/grp.rs:134-147); call before the first step."""
        _lib.check(self.L.mjx_env_enable_grp(self._h, int(max_kyoku)), "mjx_env_enable_grp")
        self._grp_cap = int(max_kyoku)

    def read_grp(self):
        """-> list (per table) of float64 [n_kyoku, 7] feature arrays, exactly dataset.Grp.take_feature() of the game's log"""
        feat = np.zeros((self.n_tables, self._grp_cap, 7), dtype=np.int32)
        cnt = np.zeros(self.n_tables, dtype=np.int32)
        _lib.check(self.L.mjx_env_read_grp(self._h, self._stream(), feat.ctypes.data, cnt.ctypes.data), "mjx_env_read_grp")
        if (cnt > self._grp_cap).any():
            raise RuntimeError(f"GRP feature overflow: {int(cnt.max())} kyoku > capacity {self._grp_cap}")
        out = []
        for t in range(self.n_tables):
            f = feat[t, : cnt[t]].astype(np.float64)
            f[:, 3:] /= 10000.0
            out.append(f)
        return out

    def set_encode_timing(self, enable: bool) -> None:
        _lib.check(self.L.mjx_env_set_encode_timing(self._h, int(enable)), "mjx_env_set_encode_timing")

    def last_encode_ms(self):
        """(k_encode_features ms, k_encode_store ms) of the last encode_obs call; needs set_encode_timing(True); blocking"""
        a, b = C.c_float(0), C.c_float(0)
        _lib.check(self.L.mjx_env_last_encode_ms(self._h, C.byref(a), C.byref(b)), "mjx_env_last_encode_ms")
        return a.value, b.value

    def launch_count(self) -> int:
        """kernels launched for this env so far (host-side counter in libmjx)"""
        return int(self.L.mjx_env_launch_count(self._h))

    def num_rows(self) -> int:
        n = C.c_int(0)
        _lib.check(self.L.mjx_env_num_rows(self._h, self._stream(), C.byref(n)), "mjx_env_num_rows")
        return n.value

    def poll(self):
        """(rows of the last step, live tables, failed tables so far, SP arena overflows so far) in one read-back"""
        out = (C.c_int * 4)()
        _lib.check(self.L.mjx_env_poll(self._h, self._stream(), out), "mjx_env_poll")
        return out[0], out[1], out[2], out[3]

    def num_live(self) -> int:
        n = C.c_int(0)
        _lib.check(self.L.mjx_env_num_live(self._h, self._stream(), C.byref(n)), "mjx_env_num_live")
        return n.value

    def total_steps(self) -> int:
        n = C.c_int64(0)
        _lib.check(self.L.mjx_env_total_steps(self._h, self._stream(), C.byref(n)), "mjx_env_total_steps")
        return n.value

    def policy_test(self, kind: int, actions, trace=None, q_values=None) -> None:
        tp = C.c_void_p(trace.data_ptr()) if trace is not None else None
        qp = C.c_void_p(q_values.data_ptr()) if q_values is not None else None
        _lib.check(self.L.mjx_env_policy_test(self._h, kind, C.c_void_p(actions.data_ptr()), tp, qp, self._stream()),
                   "mjx_env_policy_test")

    def results(self):
        n = self.n_tables
        scores = np.zeros((n, 4), dtype=np.int32)
        ranks = np.zeros((n, 4), dtype=np.uint8)
        steps = np.zeros(n, dtype=np.int32)
        err = np.zeros(n, dtype=np.int32)
        done = np.zeros(n, dtype=np.int32)
        _lib.check(self.L.mjx_env_results(self._h, self._stream(), scores.ctypes.data, ranks.ctypes.data,
                                          steps.ctypes.data, err.ctypes.data, done.ctypes.data), "mjx_env_results")
        return dict(scores=scores, ranks=ranks, steps=steps, err=err, done=done)

    def run_test_policy(self, kind: int = 1, *, encode_obs: bool = False, max_cycles: int = 0, trace: bool = False,
                        agari_guard: bool = False):
        """Play every table to the end with the built-in counter-based test policy (env-only loop)."""
        torch = self.torch
        actions = torch.zeros(self.row_cap, dtype=torch.int64, device=self.device)
        q = None
        if agari_guard:
            self.set_agari_guard(np.ones((self.n_tables, 4), dtype=np.uint8))
            q = torch.zeros((self.row_cap, 46), dtype=torch.float32, device=self.device)
        tbuf = torch.zeros((self.row_cap, 6), dtype=torch.int64, device=self.device) if trace else None
        traces = []
        cycles = 0
        first = True
        while True:
            self.step(None if first else actions, None if first else q)
            first = False
            if encode_obs:
                self.encode_obs()
            self.policy_test(kind, actions, tbuf, q)
            cycles += 1
            if trace:
                n = self.num_rows()
                traces.append(tbuf[:n].cpu().numpy().copy())
                if self.num_live() == 0:
                    break
            elif cycles % 16 == 0 and self.num_live() == 0:
                break
            if max_cycles and cycles >= max_cycles:
                break
        res = self.results()
        res["cycles"] = cycles
        if trace:
            res["trace"] = np.concatenate(traces) if traces else np.zeros((0, 6), dtype=np.int64)
        return res


class ReplayEnv(BatchEnv):
    """Replay mode (include/mjx.h mjx_env_create_replay): jobs = (game log, player) pairs advanced from logged decision to
    logged decision; the encoder API of BatchEnv applies unchanged. `jobs` comes from mortal_b200.dataset_codec.build_jobs, or
    has `hdr` and `kyoku` as int64 CUDA tensors of `device` (the decoder's arrays; mjx_env_create_replay_dev)."""

    def __init__(self, jobs, *, obs_version: int = 4, always_include_kan_select: bool = True, device: int = 0):
        import torch

        if not torch.cuda.is_available():
            raise _lib.MjxError("mortal_b200.ReplayEnv needs a CUDA device (there is no CPU fallback)")
        self.torch = torch
        self.device = torch.device("cuda", device)
        torch.cuda.set_device(self.device)
        _lib.init(device)
        self.L = _lib.load()
        on_dev = isinstance(jobs["hdr"], torch.Tensor)  # hdr / kyoku already on the device (mjx_env_create_replay_dev)
        j = {k: v if on_dev and k in ("hdr", "kyoku") else np.ascontiguousarray(v) for k, v in jobs.items()}
        self.n_tables = int(len(j["players"]))
        self.obs_version = obs_version
        self.obs_rows = self.L.mjx_obs_rows(obs_version)
        h = C.c_void_p()
        if on_dev:
            hdr, ky = j["hdr"].contiguous(), j["kyoku"].contiguous()
            _lib.check(self.L.mjx_env_create_replay_dev(C.byref(h), self.n_tables, hdr.data_ptr(), j["ev_off"].ctypes.data,
                                                        j["ev_cnt"].ctypes.data, hdr.numel(), ky.data_ptr() if ky.numel() else None,
                                                        j["ky_off"].ctypes.data, ky.numel(), j["players"].ctypes.data, obs_version,
                                                        int(always_include_kan_select), torch.cuda.current_stream(self.device).cuda_stream),
                       "mjx_env_create_replay_dev")
        else:
            _lib.check(self.L.mjx_env_create_replay(C.byref(h), self.n_tables, j["hdr"].ctypes.data, j["ev_off"].ctypes.data,
                                                    j["ev_cnt"].ctypes.data, len(j["hdr"]), j["kyoku"].ctypes.data,
                                                    j["ky_off"].ctypes.data, len(j["kyoku"]), j["players"].ctypes.data, obs_version,
                                                    int(always_include_kan_select)), "mjx_env_create_replay")
        self._h = h
        self._bind_views()
        self.row_label = self._as_t(self.L.mjx_env_row_label(h), (self.row_cap,), "<i8")
        self.row_meta = self._as_t(self.L.mjx_env_row_meta(h), (self.row_cap, 4), "|u1")

    def trust_seeds(self, nonces, keys, shuffle_kind: int = 0) -> None:
        """Per-job game seeds (start_game.seed): walls are regenerated on device, which the invisible observation needs."""
        n_ = np.ascontiguousarray(nonces, dtype=np.uint64)
        k_ = np.ascontiguousarray(keys, dtype=np.uint64)
        assert n_.shape == k_.shape == (self.n_tables,)
        _lib.check(self.L.mjx_env_replay_trust_seeds(self._h, n_.ctypes.data, k_.ctypes.data, shuffle_kind), "mjx_env_replay_trust_seeds")

    def viewpoints(self) -> None:
        """Single-viewpoint logs (mjx_env_replay_viewpoints): a job whose log hides other seats' tiles (`?` haipai or tsumo) replays
        from its player's own PlayerState, and fails with error code 13 when it hides the player's own tiles. Full-information logs
        replay exactly as without the call. Call before the first replay_step; not together with trust_seeds."""
        _lib.check(self.L.mjx_env_replay_viewpoints(self._h, self._stream()), "mjx_env_replay_viewpoints")

    def replay_step(self) -> None:
        _lib.check(self.L.mjx_env_replay_step(self._h, self._stream()), "mjx_env_replay_step")
