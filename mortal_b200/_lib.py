"""ctypes loader for mortal_b200/libmjx.so (the C ABI declared in include/mjx.h)."""
from __future__ import annotations

import ctypes as C
import os

from . import _cdecl

HERE = os.path.dirname(os.path.abspath(__file__))
DATA_DIR = os.path.join(HERE, "data")
_LIB = None
_INIT_DEVICE = None


class MjxError(RuntimeError):
    pass


def lib_path() -> str:
    return os.path.join(HERE, "libmjx.so")


class AgariIn(C.Structure):
    _fields_ = [
        ("tehai", C.c_uint8 * 34),
        ("chis", C.c_uint8 * 4), ("pons", C.c_uint8 * 4), ("minkans", C.c_uint8 * 4), ("ankans", C.c_uint8 * 4),
        ("n_chis", C.c_uint8), ("n_pons", C.c_uint8), ("n_minkans", C.c_uint8), ("n_ankans", C.c_uint8),
        ("bakaze", C.c_uint8), ("jikaze", C.c_uint8), ("winning_tile", C.c_uint8), ("is_ron", C.c_uint8),
        ("additional_hans", C.c_uint8), ("doras", C.c_uint8), ("is_oya", C.c_uint8), ("pad", C.c_uint8),
    ]


class AgariOut(C.Structure):
    _fields_ = [("kind", C.c_uint8), ("fu", C.c_uint8), ("han", C.c_uint8), ("yakuman", C.c_uint8),
                ("ron", C.c_int32), ("tsumo_ko", C.c_int32), ("tsumo_oya", C.c_int32)]


# every function include/mjx.h declares: {name: (restype, argtypes)}
SYMBOLS = _cdecl.functions(_cdecl.header(), "mjx_")


def load():
    """Load libmjx.so and bind every function include/mjx.h declares. Fails loudly if the library was not built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if not os.path.exists(path):
        raise MjxError(f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(nvcc, sm_90a). mortal_b200 has no CPU fallback.")
    _LIB = _cdecl.bind(C.CDLL(path), SYMBOLS)
    return _LIB


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().mjx_last_error()
        raise MjxError(f"{what}: {msg.decode() if msg else rc}")


def init(device: int = 0) -> None:
    """mjx_init: upload the lookup tables to `device` (idempotent)."""
    global _INIT_DEVICE
    L = load()
    if _INIT_DEVICE == device:
        return
    check(L.mjx_init(DATA_DIR.encode(), device), "mjx_init")
    _INIT_DEVICE = device
