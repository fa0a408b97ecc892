"""mortal_b200 — H100-native batched riichi-mahjong self-play environment.

Drop-in for the self-play hot path of Equim-chan/Mortal's `libriichi` (arena.OneVsThree ->
BatchGame::run -> PlayerState.update / encode_obs). The compute lives in hand-written sm_90a CUDA
kernels behind the C ABI of include/mjx.h (mortal_b200/libmjx.so); this package is the thin Python
host layer that mirrors libriichi's Python surface. There is no CPU implementation in this
package: importing works anywhere, but every compute call requires the CUDA library and a GPU.
"""
from ._lib import MjxError, lib_path, load  # noqa: F401
from .env import BatchEnv, ReplayEnv  # noqa: F401

__all__ = ["BatchEnv", "ReplayEnv", "MjxError", "load", "lib_path"]
