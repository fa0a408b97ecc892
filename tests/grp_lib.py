"""Helpers of the GRP tests — TEST INFRASTRUCTURE: the host build of csrc/mjx_grp.cuh (tests/host_emul/emul_grp.cc), the arrays
k_grp_logs reads (stat_lib.encode: the decoder's layout, encoded on the host), and the host path's per-log expectation."""
from __future__ import annotations

import numpy as np

import emul_lib as E
import stat_lib as S
from mortal_b200 import _cdecl
from mortal_b200.dataset import Grp

STATUS = {v: k.removeprefix("MJX_GRP_") for k, v in _cdecl.enum(_cdecl.header(), "mjx_grp_status").items()}  # code -> name
encode = S.encode


def run_emul(a, n_hdr=None, n_kyoku_words=None):
    """the emulated kernel over encode()'s arrays -> (feat int32 [n_kyoku, 7], rank uint8 [n, 4], final int64 [n, 4], status int32 [n]);
    n_hdr / n_kyoku_words override the capacities (hostile-array tests)"""
    L = E.lib()
    n = len(a["ev_off"])
    nk = len(a["kyoku"]) if n_kyoku_words is None else n_kyoku_words
    feat = np.full((max(nk // 19, 1), 7), -1, dtype=np.int32)
    rank = np.full((n, 4), 255, dtype=np.uint8)
    final = np.full((n, 4), -1, dtype=np.int64)
    status = np.full(n, -1, dtype=np.int32)
    ptr = lambda x: x.ctypes.data if x.size else None
    rc = L.emulg_grp_logs(n, ptr(a["hdr"]), a["ev_off"].ctypes.data, a["ev_cnt"].ctypes.data, len(a["hdr"]) if n_hdr is None else n_hdr,
                          ptr(a["kyoku"]), a["ky_off"].ctypes.data, nk, ptr(a["deltas"]), ptr(a["has"]), feat.ctypes.data,
                          rank.ctypes.data, final.ctypes.data, status.ctypes.data)
    assert rc == 0
    return feat[:nk // 19], rank, final, status


def grp_of(a, out, i):
    """log i's Grp from run_emul's outputs the way mortal_b200.dataset builds it, or None for a non-zero status"""
    feat, rank, final, status = out
    if status[i] != 0:
        return None
    lo = int(a["ky_off"][i])
    n_ky = (int(a["ky_off"][i + 1]) if i + 1 < len(a["ky_off"]) else len(feat)) - lo
    f = feat[lo:lo + n_ky].astype(np.float64)
    f[:, 3:] /= 10000.0
    return Grp(f, rank[i].tolist(), final[i].tolist())


def host_grp(events):
    """Grp.load_events, or the exception type it raises"""
    try:
        return Grp.load_events(events)
    except Exception as e:  # noqa: BLE001
        return type(e)


def same(a, b) -> bool:
    return (a.take_feature().shape == b.take_feature().shape and np.array_equal(a.take_feature(), b.take_feature())
            and a.take_feature().dtype == b.take_feature().dtype and a.take_rank_by_player() == b.take_rank_by_player()
            and a.take_final_scores() == b.take_final_scores())
