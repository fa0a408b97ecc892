"""mjai events -> the compact event words the replay kernel consumes (the inverse of mortal_b200.mjai_log.decode_events;
word layout in csrc/mjx_step.cuh `log_word`, job layout in csrc/mjx_replay.cuh)."""
from __future__ import annotations

import json

import numpy as np

from .mjai_log import (ANKAN, CHI, DAHAI, DAIMINKAN, DORA, END_KYOKU, HORA, KAKAN, PON, REACH, REACH_ACCEPTED, RYUKYOKU,
                       START_KYOKU, TILE_NAMES, TSUMO)

START_GAME, END_GAME = 15, 16
TILE_ID = {name: i for i, name in enumerate(TILE_NAMES)}
_TYPES = {"start_kyoku": START_KYOKU, "tsumo": TSUMO, "dahai": DAHAI, "chi": CHI, "pon": PON, "daiminkan": DAIMINKAN,
          "kakan": KAKAN, "ankan": ANKAN, "dora": DORA, "reach": REACH, "reach_accepted": REACH_ACCEPTED, "hora": HORA,
          "ryukyoku": RYUKYOKU, "end_kyoku": END_KYOKU, "start_game": START_GAME, "end_game": END_GAME}


def _word(ty, actor=0, target=0, pai=37, tsumogiri=0, c=(0, 0, 0, 0)):
    return (ty | (actor & 3) << 8 | (target & 3) << 10 | (pai & 0xFF) << 12 | (tsumogiri & 1) << 20
            | c[0] << 24 | c[1] << 32 | c[2] << 40 | c[3] << 48)


KYOKU_WORDS = 19  # csrc/mjx_replay.cuh REPLAY_KYOKU_WORDS: 2 score words + the 136-byte wall (17 words)


HORA_WORDS = 2  # include/mjx.h MJX_HORA_WORDS


def _hora_entry(ev, t):
    """the facts of a hora the event word drops and bin/validate_logs.rs checks (include/mjx.h, mjx_validate_logs)"""
    deltas, ura = ev.get("deltas"), ev.get("ura_markers")
    w0 = (0 if deltas is None else int(deltas[ev["actor"]]) & 0xFFFFFFFF) | int(deltas is not None) << 32 | int(ura is not None) << 33
    w1 = 0
    if ura is not None:
        w0 |= min(len(ura), 15) << 36
        for k, x in enumerate(ura[:5]):
            w1 |= t[x] << (8 * k)
    return [w0, w1]


def encode_events(events, walls=None, hora=None):
    """events: list of mjai dicts (a whole game, start_game .. end_game) -> (header words uint64 [n], kyoku payload uint64 [k, 19]).
    walls: optional uint8 [k, 136] (board.rs:109-122 layout) — the hidden tiles of every kyoku for the invisible observation;
    without them only the 52 dealt tiles are known and the rest of the wall is `?`.
    hora: optional list; every hora event appends its HORA_WORDS-word side entry (deltas[actor], ura markers) to it."""
    hdr, pay = [], []
    for ev in events:
        ty = _TYPES[ev["type"]]
        t = TILE_ID
        if ty == START_KYOKU:
            kyoku_abs = (t[ev["bakaze"]] - 27) * 4 + ev["kyoku"] - 1
            hdr.append(_word(ty, pai=t[ev["dora_marker"]], c=(kyoku_abs, ev["honba"], ev["kyotaku"], ev["oya"])))
            sc = [int(x) & 0xFFFFFFFF for x in ev["scores"]]
            flat = bytearray(t[x] for hand in ev["tehais"] for x in hand) + bytearray([37] * 84)
            if walls is not None:
                w = bytes(walls[len(pay)])
                if bytes(flat[:52]) != w[:52]:
                    raise ValueError("the wall given for a kyoku does not start with its logged haipai")
                flat = bytearray(w)
            pay.append([sc[0] | sc[1] << 32, sc[2] | sc[3] << 32] + [int.from_bytes(flat[8 * k:8 * k + 8], "little") for k in range(17)])
        elif ty in (TSUMO,):
            hdr.append(_word(ty, ev["actor"], pai=t[ev["pai"]]))
        elif ty == DAHAI:
            hdr.append(_word(ty, ev["actor"], pai=t[ev["pai"]], tsumogiri=int(ev["tsumogiri"])))
        elif ty in (CHI, PON, DAIMINKAN):
            cons = [t[x] for x in ev["consumed"]] + [37] * (4 - len(ev["consumed"]))
            hdr.append(_word(ty, ev["actor"], ev["target"], t[ev["pai"]], c=cons))
        elif ty == KAKAN:
            cons = [t[x] for x in ev["consumed"]] + [37]
            hdr.append(_word(ty, ev["actor"], pai=t[ev["pai"]], c=cons))
        elif ty == ANKAN:
            hdr.append(_word(ty, ev["actor"], c=[t[x] for x in ev["consumed"]]))
        elif ty == DORA:
            hdr.append(_word(ty, pai=t[ev["dora_marker"]]))
        elif ty in (REACH, REACH_ACCEPTED):
            hdr.append(_word(ty, ev["actor"]))
        elif ty == HORA:
            hdr.append(_word(ty, ev["actor"], ev["target"]))
            if hora is not None:
                hora.append(_hora_entry(ev, t))
        else:  # ryukyoku, end_kyoku, start_game, end_game
            hdr.append(_word(ty))
    return np.array(hdr, dtype=np.uint64), np.array(pay, dtype=np.uint64).reshape(-1, KYOKU_WORDS)


_ACTOR_FIELDS = {"tsumo": ("actor",), "dahai": ("actor",), "chi": ("actor", "target"), "pon": ("actor", "target"),
                 "daiminkan": ("actor", "target"), "kakan": ("actor",), "ankan": ("actor",), "reach": ("actor",),
                 "reach_accepted": ("actor",), "hora": ("actor", "target"), "start_kyoku": ("oya",)}
_TILE_FIELDS = {"start_kyoku": ("bakaze", "dora_marker"), "tsumo": ("pai",), "dahai": ("pai",), "chi": ("pai",), "pon": ("pai",),
                "daiminkan": ("pai",), "kakan": ("pai",), "dora": ("dora_marker",)}
_CONSUMED = {"chi": 2, "pon": 2, "daiminkan": 3, "kakan": 3, "ankan": 4}


def _is_int(x, lo, hi):
    return isinstance(x, int) and not isinstance(x, bool) and lo <= x <= hi


def check_event(ev):
    """The structural checks deserialising an mjai Event makes (mjai/event.rs:20-120): None when `ev` is well formed, else the
    name of the first failed check (the PARSE reasons of include/mjx.h). Unknown extra fields (such as `meta`) are ignored;
    a missing `deltas` / `ura_markers` on a hora is not a parse error (bin/validate_logs.rs checks it)."""
    if not isinstance(ev, dict):
        return "json"
    ty = ev.get("type")
    if not isinstance(ty, str) or ty not in _TYPES:
        return "unknown type"
    for f in _ACTOR_FIELDS.get(ty, ()):
        if f not in ev:
            return "missing or invalid field"
        if not _is_int(ev[f], 0, 3):
            return "actor out of range"
    for f in _TILE_FIELDS.get(ty, ()):
        if f not in ev:
            return "missing or invalid field"
        if ev[f] not in TILE_ID:
            return "unknown tile"
    if ty in _CONSUMED:
        c = ev.get("consumed")
        if not isinstance(c, list):
            return "missing or invalid field"
        if len(c) != _CONSUMED[ty]:
            return "consumed length"
        if any(not isinstance(x, str) or x not in TILE_ID for x in c):
            return "unknown tile"
    if ty == "dahai" and not isinstance(ev.get("tsumogiri"), bool):
        return "missing or invalid field"
    if ty == "start_kyoku":
        if not (_is_int(ev.get("kyoku"), 1, 4) and _is_int(ev.get("honba"), 0, 255) and _is_int(ev.get("kyotaku"), 0, 255)):
            return "missing or invalid field"
        sc = ev.get("scores")
        if not (isinstance(sc, list) and len(sc) == 4 and all(_is_int(x, -2**31, 2**31 - 1) for x in sc)):
            return "missing or invalid field"
        th = ev.get("tehais")
        if not (isinstance(th, list) and len(th) == 4 and all(isinstance(h, list) and len(h) == 13 for h in th)):
            return "missing or invalid field"
        if any(not isinstance(x, str) or x not in TILE_ID for h in th for x in h):
            return "unknown tile"
    if ty in ("hora", "ryukyoku") and ev.get("deltas") is not None:
        d = ev["deltas"]
        if not (isinstance(d, list) and len(d) == 4 and all(_is_int(x, -2**31, 2**31 - 1) for x in d)):
            return "missing or invalid field"
    if ty == "hora" and ev.get("ura_markers") is not None:
        u = ev["ura_markers"]
        if not isinstance(u, list):
            return "missing or invalid field"
        if any(not isinstance(x, str) or x not in TILE_ID for x in u):
            return "unknown tile"
    return None


def _swap_tile(name: str) -> str:
    """tile.rs:154-167 Tile::augment: manzu <-> pinzu, red fives stay red, souzu / honours / unknown unchanged"""
    if len(name) >= 2 and name[0].isdigit() and name[1] in "mp":
        return name[0] + ("p" if name[1] == "m" else "m") + name[2:]
    return name


def augment_events(events):
    """mjai/event.rs:187-217 Event::augment applied to a whole game: returns new event dicts, the input is not modified"""
    out = []
    for ev in events:
        e = dict(ev)
        for key in ("pai", "dora_marker", "bakaze"):
            if key in e:
                e[key] = _swap_tile(e[key])
        if "consumed" in e:
            e["consumed"] = [_swap_tile(x) for x in e["consumed"]]
        if "tehais" in e:
            e["tehais"] = [[_swap_tile(x) for x in hand] for hand in e["tehais"]]
        if e.get("ura_markers") is not None:
            e["ura_markers"] = [_swap_tile(x) for x in e["ura_markers"]]
        out.append(e)
    return out


def parse_log(text: str):
    return [json.loads(ln) for ln in text.splitlines() if ln.strip()]


def new_unknown_tiles():
    """dataset/invisible.rs:234-243"""
    u = [4] * 37
    u[4] = u[13] = u[22] = 3
    u[34] = u[35] = u[36] = 1
    return u


def reconstruct_walls(events, rng):
    """dataset/invisible.rs:24-148 Invisible::new without `trust_seed`: what the log shows of every kyoku's hidden tiles (live wall
    in drawing order, rinshan, dora and ura indicators), the rest filled with the unseen tiles in random order (the reference
    uses thread_rng there; `rng` is a numpy Generator) -> uint8 [n_kyoku, 136] in the board.rs:109-122 layout."""
    t = TILE_ID
    walls = []
    cur = None
    for ev in events:
        ty = ev["type"]
        if ty == "start_kyoku":
            cur = dict(yama=[], rinshan=[], dora=[t[ev["dora_marker"]]], ura=[], tehais=[[t[x] for x in hand] for hand in ev["tehais"]],
                       from_rinshan=False, ura_recorded=False, unknown=new_unknown_tiles())
            cur["unknown"][t[ev["dora_marker"]]] -= 1
            for hand in cur["tehais"]:
                for x in hand:
                    cur["unknown"][x] -= 1
        elif cur is None:
            continue
        elif ty == "tsumo":
            (cur["rinshan"] if cur["from_rinshan"] else cur["yama"]).append(t[ev["pai"]])
            cur["from_rinshan"] = False
            if len(cur["yama"]) > 70:
                raise ValueError("yama size overflow")
            cur["unknown"][t[ev["pai"]]] -= 1
        elif ty in ("ankan", "kakan", "daiminkan"):
            cur["from_rinshan"] = True
        elif ty == "dora":
            cur["dora"].append(t[ev["dora_marker"]])
            cur["unknown"][t[ev["dora_marker"]]] -= 1
        elif ty == "hora" and ev.get("ura_markers") is not None and not cur["ura_recorded"]:
            for x in ev["ura_markers"]:
                cur["ura"].append(t[x])
                cur["unknown"][t[x]] -= 1
            cur["ura_recorded"] = True
        elif ty == "end_kyoku":
            filler = [tid for tid, cnt in enumerate(cur["unknown"]) for _ in range(max(cnt, 0))]
            filler = [filler[i] for i in rng.permutation(len(filler))]
            for key, size in (("yama", 70), ("rinshan", 4), ("dora", 5), ("ura", 5)):
                while len(cur[key]) < size:
                    cur[key].append(filler.pop())
            if filler:
                raise ValueError("inconsistent log: more unseen tiles than hidden slots")
            w = np.zeros(136, dtype=np.uint8)
            for s_, hand in enumerate(cur["tehais"]):
                w[13 * s_:13 * s_ + 13] = hand
            for i, x in enumerate(cur["yama"]):
                w[135 - i] = x
            for i, x in enumerate(cur["rinshan"]):
                w[55 - i] = x
            for i, x in enumerate(cur["dora"]):
                w[60 - i] = x
            for i, x in enumerate(cur["ura"]):
                w[61 + i] = x
            walls.append(w)
            cur = None
    return np.stack(walls) if walls else np.zeros((0, 136), dtype=np.uint8)


def build_jobs(games, players_per_game, walls_per_game=None):
    """games: list of event lists; players_per_game: list of player-id lists -> concatenated arrays for the replay kernels"""
    hdrs, pays, ev_off, ev_cnt, ky_off, players, job_game = [], [], [], [], [], [], []
    n_hdr = n_pay = 0
    for g, (events, pids) in enumerate(zip(games, players_per_game)):
        h, p = encode_events(events, None if walls_per_game is None else walls_per_game[g])
        for pid in pids:
            ev_off.append(n_hdr); ev_cnt.append(len(h)); ky_off.append(n_pay); players.append(pid); job_game.append(g)
        hdrs.append(h); pays.append(p)
        n_hdr += len(h); n_pay += len(p)
    cat = lambda xs, shape: np.concatenate(xs) if xs else np.zeros(shape, dtype=np.uint64)
    return dict(hdr=cat(hdrs, (0,)), kyoku=cat(pays, (0, KYOKU_WORDS)).reshape(-1), ev_off=np.array(ev_off, dtype=np.int32),
                ev_cnt=np.array(ev_cnt, dtype=np.int32), ky_off=np.array(ky_off, dtype=np.int32),
                players=np.array(players, dtype=np.uint8), job_game=np.array(job_game, dtype=np.int32))
