"""ctypes binding of oracle/liboracle.so — TEST INFRASTRUCTURE (never imported by mortal_b200/)."""
from __future__ import annotations

import ctypes as C
import json
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
DATA_DIR = os.path.join(ROOT, "mortal_b200", "data")

TILE_NAMES = (
    [f"{i}m" for i in range(1, 10)] + [f"{i}p" for i in range(1, 10)] + [f"{i}s" for i in range(1, 10)]
    + ["E", "S", "W", "N", "P", "F", "C", "5mr", "5pr", "5sr", "?"]
)
TILE_ID = {n: i for i, n in enumerate(TILE_NAMES)}

EV = dict(none=0, start_game=1, start_kyoku=2, tsumo=3, dahai=4, chi=5, pon=6, daiminkan=7, kakan=8, ankan=9,
          dora=10, reach=11, reach_accepted=12, hora=13, ryukyoku=14, end_kyoku=15, end_game=16)
EV_NAME = {v: k for k, v in EV.items()}


class OrcEvent(C.Structure):
    _fields_ = [
        ("type", C.c_uint8), ("actor", C.c_uint8), ("target", C.c_uint8), ("pai", C.c_uint8), ("tsumogiri", C.c_uint8),
        ("consumed", C.c_uint8 * 4),
        ("bakaze", C.c_uint8), ("kyoku", C.c_uint8), ("honba", C.c_uint8), ("kyotaku", C.c_uint8), ("oya", C.c_uint8),
        ("scores", C.c_int32 * 4),
        ("tehais", (C.c_uint8 * 13) * 4),
        ("has_deltas", C.c_uint8),
        ("deltas", C.c_int32 * 4),
        ("ura_markers", C.c_uint8 * 5),
        ("n_ura", C.c_uint8),
    ]


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


AGARI_IN_DTYPE = np.dtype([
    ("tehai", "u1", 34), ("chis", "u1", 4), ("pons", "u1", 4), ("minkans", "u1", 4), ("ankans", "u1", 4),
    ("n_chis", "u1"), ("n_pons", "u1"), ("n_minkans", "u1"), ("n_ankans", "u1"),
    ("bakaze", "u1"), ("jikaze", "u1"), ("winning_tile", "u1"), ("is_ron", "u1"),
    ("additional_hans", "u1"), ("doras", "u1"), ("is_oya", "u1"), ("pad", "u1"),
])
AGARI_OUT_DTYPE = np.dtype([("kind", "u1"), ("fu", "u1"), ("han", "u1"), ("yakuman", "u1"),
                            ("ron", "<i4"), ("tsumo_ko", "<i4"), ("tsumo_oya", "<i4")])
assert AGARI_IN_DTYPE.itemsize == C.sizeof(AgariIn) == 62
assert AGARI_OUT_DTYPE.itemsize == C.sizeof(AgariOut) == 16


class PsView(C.Structure):
    _fields_ = [
        ("tehai", C.c_uint8 * 34), ("waits", C.c_uint8 * 34), ("dora_factor", C.c_uint8 * 34),
        ("tiles_seen", C.c_uint8 * 34), ("keep_shanten_discards", C.c_uint8 * 34),
        ("next_shanten_discards", C.c_uint8 * 34), ("forbidden_tiles", C.c_uint8 * 34),
        ("discarded_tiles", C.c_uint8 * 34),
        ("akas_seen", C.c_uint8 * 3), ("akas_in_hand", C.c_uint8 * 3),
        ("bakaze", C.c_uint8), ("jikaze", C.c_uint8), ("kyoku", C.c_uint8), ("honba", C.c_uint8),
        ("kyotaku", C.c_uint8), ("rank", C.c_uint8), ("oya", C.c_uint8), ("is_all_last", C.c_uint8),
        ("scores", C.c_int32 * 4),
        ("n_dora_indicators", C.c_uint8), ("dora_indicators", C.c_uint8 * 5),
        ("riichi_declared", C.c_uint8 * 4), ("riichi_accepted", C.c_uint8 * 4),
        ("at_turn", C.c_uint8), ("tiles_left", C.c_uint8),
        ("shanten", C.c_int8), ("real_time_shanten", C.c_int8),
        ("has_last_self_tsumo", C.c_uint8), ("last_self_tsumo", C.c_uint8),
        ("has_last_kawa_tile", C.c_uint8), ("last_kawa_tile", C.c_uint8),
        ("cans", C.c_uint32),
        ("n_ankan_candidates", C.c_uint8), ("ankan_candidates", C.c_uint8 * 3),
        ("n_kakan_candidates", C.c_uint8), ("kakan_candidates", C.c_uint8 * 3),
        ("chankan_chance", C.c_uint8), ("can_w_riichi", C.c_uint8), ("is_w_riichi", C.c_uint8),
        ("at_rinshan", C.c_uint8), ("at_ippatsu", C.c_uint8), ("at_furiten", C.c_uint8),
        ("to_mark_same_cycle_furiten", C.c_uint8), ("kans_on_board", C.c_uint8), ("is_menzen", C.c_uint8),
        ("n_chis", C.c_uint8), ("chis", C.c_uint8 * 4), ("n_pons", C.c_uint8), ("pons", C.c_uint8 * 4),
        ("n_minkans", C.c_uint8), ("minkans", C.c_uint8 * 4), ("n_ankans", C.c_uint8), ("ankans", C.c_uint8 * 4),
        ("doras_owned", C.c_uint8 * 4), ("doras_seen", C.c_uint8), ("tehai_len_div3", C.c_uint8),
        ("has_next_shanten_discard", C.c_uint8),
        ("kawa_len", C.c_uint8 * 4),
    ]


class SpIn(C.Structure):
    _fields_ = [
        ("tehai", C.c_uint8 * 34), ("akas_in_hand", C.c_uint8 * 3), ("tiles_seen", C.c_uint8 * 34),
        ("akas_seen", C.c_uint8 * 3),
        ("tehai_len_div3", C.c_uint8), ("is_menzen", C.c_uint8), ("bakaze", C.c_uint8), ("jikaze", C.c_uint8),
        ("num_doras_in_fuuro", C.c_uint8),
        ("n_dora_indicators", C.c_uint8), ("dora_indicators", C.c_uint8 * 5),
        ("calc_double_riichi", C.c_uint8), ("calc_haitei", C.c_uint8), ("prefer_riichi", C.c_uint8),
        ("sort_result", C.c_uint8), ("maximize_win_prob", C.c_uint8), ("calc_tegawari", C.c_uint8),
        ("calc_shanten_down", C.c_uint8),
        ("chis", C.c_uint8 * 4), ("pons", C.c_uint8 * 4), ("minkans", C.c_uint8 * 4), ("ankans", C.c_uint8 * 4),
        ("n_chis", C.c_uint8), ("n_pons", C.c_uint8), ("n_minkans", C.c_uint8), ("n_ankans", C.c_uint8),
        ("can_discard", C.c_uint8), ("tsumos_left", C.c_uint8), ("cur_shanten", C.c_int8),
    ]


class SpCand(C.Structure):
    _fields_ = [
        ("tile", C.c_uint8), ("shanten_down", C.c_uint8), ("num_required_tiles", C.c_uint8),
        ("n_required", C.c_uint8), ("n_turns", C.c_uint8),
        ("required_tile", C.c_uint8 * 34), ("required_count", C.c_uint8 * 34),
        ("tenpai_probs", C.c_float * 17), ("win_probs", C.c_float * 17), ("exp_values", C.c_float * 17),
    ]


class RunCfg(C.Structure):
    _fields_ = [("n_tables", C.c_int32), ("shuffle_kind", C.c_int32), ("policy_kind", C.c_int32),
                ("enable_quick_eval", C.c_int32), ("enable_agari_guard", C.c_int32), ("encode_obs", C.c_int32),
                ("sp_mode", C.c_int32), ("n_threads", C.c_int32), ("max_steps_per_table", C.c_int64),
                ("encode_from_step", C.c_int64)]


class RunOut(C.Structure):
    _fields_ = [("table_steps", C.c_int64), ("obs_rows", C.c_int64), ("seconds", C.c_double)]


_lib = None


def build(force: bool = False) -> str:
    so = os.path.join(ORACLE_DIR, "liboracle.so")
    srcs = [os.path.join(ORACLE_DIR, f) for f in os.listdir(ORACLE_DIR) if f.endswith((".cc", ".h"))] + \
        [os.path.join(ROOT, "include", "mjx.h")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", ORACLE_DIR, "liboracle.so"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _lib
    if _lib is not None:
        return _lib
    L = C.CDLL(build())
    L.orc_last_error.restype = C.c_char_p
    L.orc_init.argtypes = [C.c_char_p]
    L.orc_shanten.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.orc_agari.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.orc_point.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int32)]
    L.orc_check_ankan_after_riichi.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.orc_rankings.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_agari_key.argtypes = [C.c_void_p, C.c_void_p]
    L.orc_agari_key.restype = C.c_uint32
    L.orc_agari_lookup.argtypes = [C.c_uint32, C.c_void_p]
    L.orc_make_wall.argtypes = [C.c_uint64, C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L.orc_sha3_256.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.orc_chacha12.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.orc_ps_new.restype = C.c_void_p
    L.orc_ps_new.argtypes = [C.c_int]
    L.orc_ps_free.argtypes = [C.c_void_p]
    L.orc_ps_clone.restype = C.c_void_p
    L.orc_ps_clone.argtypes = [C.c_void_p]
    L.orc_ps_update.restype = C.c_int64
    L.orc_ps_update.argtypes = [C.c_void_p, C.POINTER(OrcEvent)]
    L.orc_ps_validate_reaction.argtypes = [C.c_void_p, C.POINTER(OrcEvent)]
    L.orc_ps_view_get.argtypes = [C.c_void_p, C.POINTER(PsView)]
    L.orc_ps_set_tehai.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.orc_ps_update_waits_and_furiten.argtypes = [C.c_void_p]
    L.orc_ps_set_can_chi_from_tile.argtypes = [C.c_void_p, C.c_int]
    L.orc_ps_set_can_chi_from_tile.restype = C.c_uint32
    L.orc_ps_get_rank.argtypes = [C.c_int, C.c_void_p]
    L.orc_ps_agari_points.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int32)]
    L.orc_ps_rule_based_agari.argtypes = [C.c_void_p]
    L.orc_ps_rule_based_agari_slow.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.orc_ps_discard_candidates.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.orc_obs_rows.argtypes = [C.c_int]
    L.orc_ps_encode_obs.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    L.orc_ps_legal_mask.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.orc_sp_calc.argtypes = [C.POINTER(SpIn), C.POINTER(SpCand), C.c_int]
    L.orc_game_new.restype = C.c_void_p
    L.orc_game_new.argtypes = [C.c_uint64, C.c_uint64, C.c_int, C.c_int]
    L.orc_game_free.argtypes = [C.c_void_p]
    L.orc_game_poll.argtypes = [C.c_void_p]
    L.orc_game_state.restype = C.c_void_p
    L.orc_game_state.argtypes = [C.c_void_p, C.c_int]
    L.orc_game_set_reaction.argtypes = [C.c_void_p, C.c_int, C.POINTER(OrcEvent)]
    L.orc_game_set_action.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.orc_game_advance_step.argtypes = [C.c_void_p]
    L.orc_game_finish.argtypes = [C.c_void_p, C.c_void_p]
    L.orc_game_info.argtypes = [C.c_void_p, C.c_void_p]
    L.orc_game_log.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.orc_gameplay_load.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 7
    L.orc_gameplay_load_oracle.argtypes = ([C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 7
                                           + [C.c_uint64, C.c_uint64, C.c_int, C.c_void_p, C.c_void_p])
    L.orc_run_batch.argtypes = [C.POINTER(RunCfg), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.POINTER(RunOut)]
    L.orc_run_replay.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p,
                                 C.c_void_p, C.c_void_p]
    L.orc_run_replay2.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                  C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_run_replay3.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                  C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_run_sample_obs.argtypes = [C.POINTER(RunCfg), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_oracle_obs_rows.argtypes = [C.c_int]
    L.orc_game_encode_oracle_obs.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    L.orc_batch_new.restype = C.c_void_p
    L.orc_batch_new.argtypes = [C.POINTER(RunCfg), C.c_void_p, C.c_void_p]
    L.orc_batch_free.argtypes = [C.c_void_p]
    L.orc_batch_run.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.POINTER(RunOut)]
    L.orc_policy_hash.restype = C.c_uint64
    L.orc_policy_hash.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32]
    if L.orc_init(DATA_DIR.encode()) != 0:
        raise RuntimeError(L.orc_last_error().decode())
    _lib = L
    return L


def err() -> str:
    return lib().orc_last_error().decode()


# ---------------------------------------------------------------- helpers
def hand_with_aka(s: str) -> np.ndarray:
    """tenhou.net/2 format (hand.rs:14-54): '0m' is the aka 5m; z = honours."""
    ret = np.zeros(37, dtype=np.uint8)
    stack = []
    for ch in s:
        if ch.isdigit():
            stack.append(int(ch))
        elif ch in "mpsz":
            for t in stack:
                if t == 0:
                    idx = {"m": 34, "p": 35, "s": 36}[ch]
                else:
                    idx = "mpsz".index(ch) * 9 + t - 1
                ret[idx] += 1
            stack = []
        elif ch in " \t\n":
            pass
        else:
            raise ValueError(ch)
    return ret


def hand(s: str) -> np.ndarray:
    h = hand_with_aka(s)
    ret = h[:34].copy()
    ret[4] += h[34]
    ret[13] += h[35]
    ret[22] += h[36]
    return ret


def tid(name: str) -> int:
    return TILE_ID[name]


def shanten(tiles: np.ndarray, len_div3, kind: int = 0) -> np.ndarray:
    tiles = np.ascontiguousarray(tiles, dtype=np.uint8).reshape(-1, 34)
    n = tiles.shape[0]
    ld = np.ascontiguousarray(np.broadcast_to(np.asarray(len_div3, dtype=np.uint8), (n,)))
    out = np.zeros(n, dtype=np.int8)
    assert lib().orc_shanten(tiles.ctypes.data, ld.ctypes.data, out.ctypes.data, n, kind) == 0, err()
    return out


def agari(queries: np.ndarray, mode: int) -> np.ndarray:
    q = np.ascontiguousarray(queries, dtype=AGARI_IN_DTYPE)
    out = np.zeros(q.shape[0], dtype=AGARI_OUT_DTYPE)
    assert lib().orc_agari(q.ctypes.data, out.ctypes.data, q.shape[0], mode) == 0, err()
    return out


def agari_query(tehai, *, chis=(), pons=(), minkans=(), ankans=(), bakaze="E", jikaze="E", winning_tile, is_ron,
                additional_hans=0, doras=0, is_oya=False) -> np.ndarray:
    q = np.zeros(1, dtype=AGARI_IN_DTYPE)
    q["tehai"][0] = hand(tehai) if isinstance(tehai, str) else tehai
    for name, v in (("chis", chis), ("pons", pons), ("minkans", minkans), ("ankans", ankans)):
        ids = [tid(x) if isinstance(x, str) else x for x in v]
        q[name][0][: len(ids)] = ids
        q["n_" + name][0] = len(ids)
    q["bakaze"] = tid(bakaze)
    q["jikaze"] = tid(jikaze)
    q["winning_tile"] = tid(winning_tile) if isinstance(winning_tile, str) else winning_tile
    q["is_ron"] = int(is_ron)
    q["additional_hans"] = additional_hans
    q["doras"] = doras
    q["is_oya"] = int(is_oya)
    return q


def event_from_json(obj) -> OrcEvent:
    """mjai JSON (dict or str) -> OrcEvent (mjai/event.rs:20-120)."""
    if isinstance(obj, str):
        obj = json.loads(obj)
    e = OrcEvent()
    e.type = EV[obj["type"]]
    e.pai = 37
    for i in range(4):
        e.consumed[i] = 37
    if "actor" in obj:
        e.actor = obj["actor"]
    if "target" in obj:
        e.target = obj["target"]
    if "pai" in obj:
        e.pai = tid(obj["pai"])
    if "dora_marker" in obj:
        e.pai = tid(obj["dora_marker"])
    if "tsumogiri" in obj:
        e.tsumogiri = int(obj["tsumogiri"])
    if "consumed" in obj:
        for i, t in enumerate(obj["consumed"]):
            e.consumed[i] = tid(t)
    if obj["type"] == "start_kyoku":
        e.bakaze = tid(obj["bakaze"])
        e.kyoku = obj["kyoku"]
        e.honba = obj["honba"]
        e.kyotaku = obj["kyotaku"]
        e.oya = obj["oya"]
        for i in range(4):
            e.scores[i] = obj["scores"][i]
            for j in range(13):
                e.tehais[i][j] = tid(obj["tehais"][i][j])
    if "deltas" in obj and obj["deltas"] is not None:
        e.has_deltas = 1
        for i in range(4):
            e.deltas[i] = obj["deltas"][i]
    if obj.get("ura_markers"):
        e.n_ura = len(obj["ura_markers"])
        for i, t in enumerate(obj["ura_markers"]):
            e.ura_markers[i] = tid(t)
    return e


def event_to_dict(e: OrcEvent) -> dict:
    t = EV_NAME[e.type]
    d = {"type": t}
    if t in ("tsumo", "dahai", "chi", "pon", "daiminkan", "kakan", "ankan", "reach", "reach_accepted", "hora"):
        d["actor"] = e.actor
    if t in ("chi", "pon", "daiminkan", "hora"):
        d["target"] = e.target
    if t in ("tsumo", "dahai", "chi", "pon", "daiminkan", "kakan"):
        d["pai"] = TILE_NAMES[e.pai]
    if t == "dahai":
        d["tsumogiri"] = bool(e.tsumogiri)
    n_cons = {"chi": 2, "pon": 2, "daiminkan": 3, "kakan": 3, "ankan": 4}.get(t, 0)
    if n_cons:
        d["consumed"] = [TILE_NAMES[e.consumed[i]] for i in range(n_cons)]
    if t == "dora":
        d["dora_marker"] = TILE_NAMES[e.pai]
    if t == "start_kyoku":
        d.update(bakaze=TILE_NAMES[e.bakaze], dora_marker=TILE_NAMES[e.pai], kyoku=e.kyoku, honba=e.honba,
                 kyotaku=e.kyotaku, oya=e.oya, scores=list(e.scores),
                 tehais=[[TILE_NAMES[e.tehais[i][j]] for j in range(13)] for i in range(4)])
    if t in ("hora", "ryukyoku") and e.has_deltas:
        d["deltas"] = list(e.deltas)
    if t == "hora":
        d["ura_markers"] = [TILE_NAMES[e.ura_markers[i]] for i in range(e.n_ura)]
    return d


CAN_BITS = ["can_discard", "can_chi_low", "can_chi_mid", "can_chi_high", "can_pon", "can_daiminkan", "can_kakan",
            "can_ankan", "can_riichi", "can_tsumo_agari", "can_ron_agari", "can_ryukyoku"]


def unpack_cans(v: int) -> dict:
    d = {name: bool((v >> i) & 1) for i, name in enumerate(CAN_BITS)}
    d["target_actor"] = (v >> 16) & 0xFF
    return d


class PlayerState:
    """Thin handle over orc::PlayerState mirroring libriichi.state.PlayerState's test-facing surface."""

    def __init__(self, player_id: int, _ptr=None, _own=True):
        self._p = _ptr if _ptr is not None else lib().orc_ps_new(player_id)
        self._own = _own

    def __del__(self):
        if getattr(self, "_own", False) and self._p:
            lib().orc_ps_free(self._p)
            self._p = None

    def clone(self) -> "PlayerState":
        return PlayerState(0, _ptr=lib().orc_ps_clone(self._p))

    def update(self, ev) -> dict:
        e = ev if isinstance(ev, OrcEvent) else event_from_json(ev)
        r = lib().orc_ps_update(self._p, C.byref(e))
        if r < 0:
            raise RuntimeError(err())
        return unpack_cans(r)

    def validate_reaction(self, ev) -> None:
        e = ev if isinstance(ev, OrcEvent) else event_from_json(ev)
        if lib().orc_ps_validate_reaction(self._p, C.byref(e)) != 0:
            raise RuntimeError(err())

    @classmethod
    def from_log(cls, player_id: int, log: str) -> "PlayerState":
        ps = cls(player_id)
        for line in log.strip().split("\n"):
            ps.update(line.strip())
        return ps

    def view(self) -> PsView:
        v = PsView()
        lib().orc_ps_view_get(self._p, C.byref(v))
        return v

    def agari_points(self, is_ron: bool, ura=()) -> dict:
        u = np.array([tid(t) if isinstance(t, str) else t for t in ura], dtype=np.uint8)
        out = (C.c_int32 * 3)()
        if lib().orc_ps_agari_points(self._p, int(is_ron), u.ctypes.data, len(u), out) != 0:
            raise RuntimeError(err())
        return dict(ron=out[0], tsumo_ko=out[1], tsumo_oya=out[2])

    def rule_based_agari(self) -> bool:
        r = lib().orc_ps_rule_based_agari(self._p)
        if r < 0:
            raise RuntimeError(err())
        return bool(r)

    def rule_based_agari_slow(self, is_ron: bool, target_rel: int) -> bool:
        r = lib().orc_ps_rule_based_agari_slow(self._p, int(is_ron), target_rel)
        if r < 0:
            raise RuntimeError(err())
        return bool(r)

    def discard_candidates(self, unconditional_tenpai: bool = False) -> np.ndarray:
        out = np.zeros(37, dtype=np.uint8)
        if lib().orc_ps_discard_candidates(self._p, int(unconditional_tenpai), out.ctypes.data) != 0:
            raise RuntimeError(err())
        return out.astype(bool)

    def encode_obs(self, version: int, at_kan_select: bool, sp_mode: int = 1):
        rows = lib().orc_obs_rows(version)
        obs = np.zeros((rows, 34), dtype=np.float32)
        mask = np.zeros(46, dtype=np.uint8)
        if lib().orc_ps_encode_obs(self._p, version, int(at_kan_select), obs.ctypes.data, mask.ctypes.data, sp_mode) != 0:
            raise RuntimeError(err())
        return obs, mask.astype(bool)

    def legal_mask(self, at_kan_select: bool = False) -> np.ndarray:
        mask = np.zeros(46, dtype=np.uint8)
        if lib().orc_ps_legal_mask(self._p, int(at_kan_select), mask.ctypes.data) != 0:
            raise RuntimeError(err())
        return mask.astype(bool)


def run_batch(nonces, keys, *, shuffle_kind=0, policy_kind=1, quick_eval=True, agari_guard=False, encode_obs=0,
              sp_mode=1, n_threads=1, max_steps=0, table_ids=None, trace_cap=0, encode_from_step=0):
    n = len(nonces)
    nonces = np.ascontiguousarray(nonces, dtype=np.uint64)
    keys = np.ascontiguousarray(keys, dtype=np.uint64)
    tids = None if table_ids is None else np.ascontiguousarray(table_ids, dtype=np.int32)
    scores = np.zeros((n, 4), dtype=np.int32)
    ranks = np.zeros((n, 4), dtype=np.uint8)
    steps = np.zeros(n, dtype=np.int32)
    trace = np.zeros((trace_cap, 6), dtype=np.int64) if trace_cap else None
    tlen = C.c_int64(0)
    cfg = RunCfg(n, shuffle_kind, policy_kind, int(quick_eval), int(agari_guard), encode_obs, sp_mode, n_threads, max_steps, encode_from_step)
    out = RunOut()
    rc = lib().orc_run_batch(C.byref(cfg), nonces.ctypes.data, keys.ctypes.data,
                             None if tids is None else tids.ctypes.data, scores.ctypes.data, ranks.ctypes.data,
                             steps.ctypes.data, None if trace is None else trace.ctypes.data, trace_cap,
                             C.byref(tlen), C.byref(out))
    if rc != 0:
        raise RuntimeError(err())
    res = dict(scores=scores, ranks=ranks, steps=steps, table_steps=out.table_steps, obs_rows=out.obs_rows,
               seconds=out.seconds)
    if trace is not None:
        assert tlen.value <= trace_cap, "trace overflow"
        res["trace"] = trace[: tlen.value]
    return res


def run_replay(nonces, keys, replay, *, shuffle_kind=0, quick_eval=True, mask_bits=None, max_steps=0, n_threads=1, quick_eval_seats=None):
    """replay: int64 [m, 5] rows (table, step, seat, kan_select, action) recorded from another implementation;
    mask_bits: optional int64 [m] legal masks the recorder saw (compared bit for bit); max_steps: the recording was cut
    after that many table-steps per table (0 = whole hanchans)."""
    n = len(nonces)
    nonces = np.ascontiguousarray(nonces, dtype=np.uint64)
    keys = np.ascontiguousarray(keys, dtype=np.uint64)
    rp = np.ascontiguousarray(replay, dtype=np.int64).reshape(-1, 5)
    order = np.lexsort((rp[:, 3], rp[:, 2], rp[:, 1], rp[:, 0]))
    rp = np.ascontiguousarray(rp[order])
    mb = None if mask_bits is None else np.ascontiguousarray(np.asarray(mask_bits, dtype=np.int64)[order])
    scores = np.zeros((n, 4), dtype=np.int32)
    ranks = np.zeros((n, 4), dtype=np.uint8)
    steps = np.zeros(n, dtype=np.int32)
    if quick_eval_seats is not None:  # uint8 [n, 4]: per-seat enable_quick_eval
        qf = np.ascontiguousarray(quick_eval_seats, dtype=np.uint8).reshape(n, 4)
        rc = lib().orc_run_replay3(n, nonces.ctypes.data, keys.ctypes.data, shuffle_kind, qf.ctypes.data, rp.ctypes.data,
                                   len(rp), None if mb is None else mb.ctypes.data, max_steps, n_threads,
                                   scores.ctypes.data, ranks.ctypes.data, steps.ctypes.data)
    else:
        rc = lib().orc_run_replay2(n, nonces.ctypes.data, keys.ctypes.data, shuffle_kind, int(quick_eval), rp.ctypes.data,
                                   len(rp), None if mb is None else mb.ctypes.data, max_steps, n_threads,
                                   scores.ctypes.data, ranks.ctypes.data, steps.ctypes.data)
    if rc != 0:
        raise RuntimeError(err())
    return dict(scores=scores, ranks=ranks, steps=steps)


def run_sample_obs(nonces, keys, samples, *, version=4, shuffle_kind=0, policy_kind=1, quick_eval=True, sp_mode=1,
                   n_threads=1, max_steps=0, invisible=False):
    """Replay the tables with the built-in counter-based policy and encode the decisions listed in `samples`
    (int64 [m, 4] rows (table, step_idx, seat, kan_select)) -> (obs f32 [m, rows, 34], masks bool [m, 46], found bool [m]),
    in the order of `samples`."""
    n = len(nonces)
    nonces = np.ascontiguousarray(nonces, dtype=np.uint64)
    keys = np.ascontiguousarray(keys, dtype=np.uint64)
    sm = np.ascontiguousarray(samples, dtype=np.int64).reshape(-1, 4)
    order = np.lexsort((sm[:, 3], sm[:, 2], sm[:, 1], sm[:, 0]))
    srt = np.ascontiguousarray(sm[order])
    m = len(srt)
    rows = {1: 938, 2: 942, 3: 934, 4: 1012}[version]
    obs = np.zeros((m, rows, 34), dtype=np.float32)
    masks = np.zeros((m, 46), dtype=np.uint8)
    found = np.zeros(m, dtype=np.uint8)
    scores = np.zeros((n, 4), dtype=np.int32)
    ranks = np.zeros((n, 4), dtype=np.uint8)
    steps = np.zeros(n, dtype=np.int32)
    cfg = RunCfg(n, shuffle_kind, policy_kind, int(quick_eval), 0, 0, sp_mode, n_threads, max_steps, 0)
    inv_obs = np.zeros((m, lib().orc_oracle_obs_rows(version), 34), dtype=np.float32) if invisible else None
    rc = lib().orc_run_sample_obs(C.byref(cfg), nonces.ctypes.data, keys.ctypes.data, scores.ctypes.data, ranks.ctypes.data,
                                  steps.ctypes.data, srt.ctypes.data, m, version, obs.ctypes.data, masks.ctypes.data,
                                  found.ctypes.data, None if inv_obs is None else inv_obs.ctypes.data)
    if rc != 0:
        raise RuntimeError(err())
    inv = np.empty(m, dtype=np.int64)
    inv[order] = np.arange(m)
    if invisible:
        return obs[inv], masks[inv].astype(bool), found[inv].astype(bool), inv_obs[inv]
    return obs[inv], masks[inv].astype(bool), found[inv].astype(bool)


def gameplay_load(events, player_id, *, version=4, always_include_kan_select=True, sp_mode=1, max_moves=2048, with_obs=True,
                  oracle_seed=None, shuffle_kind=0, walls=None):
    """dataset/gameplay.rs GameplayLoader for one (game, player): events = list of mjai dicts (start_game .. end_game).
    oracle_seed = (nonce, key): additionally the invisible observations of `oracle=True, trust_seed=True` ("invisible")."""
    evs = (OrcEvent * len(events))(*[event_from_json(e) for e in events])
    rows = {1: 938, 2: 942, 3: 934, 4: 1012}[version]
    obs = np.zeros((max_moves, rows, 34), dtype=np.float32) if with_obs else None
    masks = np.zeros((max_moves, 46), dtype=np.uint8)
    actions = np.zeros(max_moves, dtype=np.int64)
    at_kyoku = np.zeros(max_moves, dtype=np.uint8); gamma = np.zeros(max_moves, dtype=np.uint8)
    at_turns = np.zeros(max_moves, dtype=np.uint8); shantens = np.zeros(max_moves, dtype=np.int8)
    inv = None
    if walls is not None:
        walls = np.ascontiguousarray(walls, dtype=np.uint8).reshape(-1, 136)
        oracle_seed = oracle_seed or (0, 0)
    if oracle_seed is None:
        n = lib().orc_gameplay_load(evs, len(events), player_id, version, int(always_include_kan_select), sp_mode, max_moves,
                                    obs.ctypes.data if with_obs else None, masks.ctypes.data, actions.ctypes.data,
                                    at_kyoku.ctypes.data, gamma.ctypes.data, at_turns.ctypes.data, shantens.ctypes.data)
    else:
        inv = np.zeros((max_moves, lib().orc_oracle_obs_rows(version), 34), dtype=np.float32)
        n = lib().orc_gameplay_load_oracle(evs, len(events), player_id, version, int(always_include_kan_select), sp_mode, max_moves,
                                           obs.ctypes.data if with_obs else None, masks.ctypes.data, actions.ctypes.data,
                                           at_kyoku.ctypes.data, gamma.ctypes.data, at_turns.ctypes.data, shantens.ctypes.data,
                                           int(oracle_seed[0]), int(oracle_seed[1]), shuffle_kind, inv.ctypes.data,
                                           None if walls is None else walls.ctypes.data)
    assert n >= 0, err()
    return dict(invisible=None if inv is None else inv[:n], obs=obs[:n] if with_obs else None, masks=masks[:n].astype(bool), actions=actions[:n], at_kyoku=at_kyoku[:n],
                apply_gamma=gamma[:n].astype(bool), at_turns=at_turns[:n], shantens=shantens[:n])


class Batch:
    """Persistent CPU arena (bench.py --impl reference): tables live across calls; run(until) advances every live table to
    `until` table-steps and returns (table_steps advanced, rows decided, seconds)."""

    def __init__(self, nonces, keys, *, shuffle_kind=0, policy_kind=2, quick_eval=True, encode_obs=4, sp_mode=1, n_threads=1):
        nonces = np.ascontiguousarray(nonces, dtype=np.uint64)
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        cfg = RunCfg(len(nonces), shuffle_kind, policy_kind, int(quick_eval), 0, encode_obs, sp_mode, n_threads, 0, 0)
        self._h = lib().orc_batch_new(C.byref(cfg), nonces.ctypes.data, keys.ctypes.data)

    def run(self, until, encode_from=0):
        out = RunOut()
        if lib().orc_batch_run(self._h, until, encode_from, C.byref(out)) != 0:
            raise RuntimeError(err())
        return out.table_steps, out.obs_rows, out.seconds

    def close(self):
        if self._h:
            lib().orc_batch_free(self._h)
            self._h = None

    def __del__(self):
        self.close()
