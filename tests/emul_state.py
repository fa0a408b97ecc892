"""Host-emulated backend for mortal_b200.libriichi.state (TEST INFRASTRUCTURE): the surface of include/mjx.h mjx_state_* served by
tests/host_emul (the single-lane g++ build of the product's device sources). Injected with state.set_backend(); never shipped."""
import ctypes as C

import numpy as np

import emul_lib as E
from mortal_b200.libriichi.state import PlayerView


class EmulStateBackend:
    def __init__(self):
        self.L = E.lib()

    def create(self, player_ids, version=4):
        ids = np.ascontiguousarray(player_ids, dtype=np.uint8)
        return self.L.emul_state_create(len(ids), ids.ctypes.data)

    def destroy(self, h):
        self.L.emul_env_destroy(h)

    def update(self, h, words, payload):
        cans = np.zeros(len(words), dtype=np.uint32)
        self.L.emul_state_update(h, words.ctypes.data, None if payload is None else payload.ctypes.data, cans.ctypes.data)
        return cans

    def view(self, h, index):
        v = PlayerView()
        self.L.emul_state_view(h, index, C.byref(v))
        return v

    def encode(self, h, n, version, kan):
        k = np.ascontiguousarray(kan, dtype=np.uint8)
        self.L.emul_state_rows(h, k.ctypes.data)
        rows = {1: 938, 2: 942, 3: 934, 4: 1012}[version]
        obs = np.zeros((n, rows, 34), dtype=np.float32)
        self.L.emul_env_encode_obs_v(h, obs.ctypes.data, 1 if version == 4 else 0, version)
        rt = np.zeros(n, dtype=np.int32); rs = np.zeros(n, dtype=np.uint8); m = np.zeros((n, 46), dtype=np.uint8)
        self.L.emul_env_rows(h, rt.ctypes.data, rs.ctypes.data, m.ctypes.data)
        return obs, m.astype(bool)

    def query(self, h, index, what, args):
        a = np.zeros(8, dtype=np.int32)
        a[: len(args)] = args
        out = np.zeros(4, dtype=np.int32)
        self.L.emul_state_query(h, index, what, a.ctypes.data, out.ctypes.data)
        return out

    def copy(self, dst, di, src, si):
        self.L.emul_state_copy(dst, di, src, si)
