"""The fused policy-net entries of libmjx refuse misaligned pointers: each mjx_nn_* call returns MJX_ERR_ARG for a pointer off
a 16-byte boundary (the kernels read 16-byte vectors and would fault), as part of its argument checks and so before the
MJX_ERR_STATE of an uninitialised library. Runs without a GPU: the check happens in a fresh process that never calls mjx_init,
so no entry can launch anything whatever it is handed, and no pointer is dereferenced."""
import json
import os
import subprocess
import sys

C_ENTRY_CHECK = r"""
import ctypes as C, json, sys
sys.path.insert(0, sys.argv[1])
from mortal_b200 import _lib
L = _lib.load()  # never mjx_init: no entry can launch a kernel, whatever it is handed
A = 1 << 24      # an aligned address; nothing is dereferenced before the argument checks
entries = {
    "affine_mish": (L.mjx_nn_affine_mish_bf16, 4, lambda p: (*p, 8 * 34 * 64, 64, None)),
    "pool": (L.mjx_nn_pool_bf16, 3, lambda p: (*p, 8, 34, 64, None)),
    "gate_residual": (L.mjx_nn_gate_residual_bf16, 4, lambda p: (*p, 8, 34, 64, None)),
    "block_tail": (L.mjx_nn_block_tail_bf16, 11, lambda p: (*p, 8, 34, 64, 4, None)),
    "obs_to_nhwc": (L.mjx_nn_obs_to_nhwc_bf16, 2, lambda p: (*p, 8, 1012, 34, 1024, None)),
}
res = {}
for name, (fn, n, args) in entries.items():
    ptrs = [A + 4096 * i for i in range(n)]
    res[name] = {"aligned": fn(*args(ptrs)),
                 "misaligned": [fn(*args([q + (4 if j == i else 0) for j, q in enumerate(ptrs)])) for i in range(n)]}
    if name == "obs_to_nhwc":
        res[name]["obs_float_aligned"] = fn(*args([ptrs[0] + 4, ptrs[1]]))
        res[name]["misaligned"][0] = fn(*args([ptrs[0] + 2, ptrs[1]]))
print(json.dumps(res))
"""


def test_c_entries_refuse_misaligned_pointers_before_state():
    """every pointer of every entry, misaligned one at a time: MJX_ERR_ARG; all aligned: MJX_ERR_STATE (no mjx_init)"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", C_ENTRY_CHECK, root], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-3000:]
    res = json.loads(out.stdout.strip().splitlines()[-1])
    ERR_ARG, ERR_STATE = -2, -4
    for name, r in res.items():
        assert r["aligned"] == ERR_STATE, (name, r)
        assert r["misaligned"] == [ERR_ARG] * len(r["misaligned"]), (name, r)
    assert res["obs_to_nhwc"]["obs_float_aligned"] == ERR_STATE  # observations need float alignment only
