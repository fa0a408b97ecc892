"""Seeded one-mutation-per-log generator for the log-validation tests: every class turns a valid mjai log into one that
bin/validate_logs.rs rejects (the expected verdict comes from the oracle, not from here)."""
from __future__ import annotations

import json
from collections import Counter

import numpy as np

TILES = [f"{i}{s}" for s in "mps" for i in range(1, 10)] + list("ESWNPFC")
AKA = {"5mr": "5m", "5pr": "5p", "5sr": "5s"}
CLASSES = ("dahai_not_held", "dahai_illegal_held", "chi_non_kamicha", "call_cannot", "riichi_not_tenpai", "hora_non_winning",
           "deltas_lowered", "hora_field_removed", "tsumo_fifth", "haipai_unknown", "unparsable")


def deaka(t: str) -> str:
    return AKA.get(t, t)


def track(events):
    """per event index: (hands [4] Counter, seen-by-everyone Counter, riichi-accepted seats) BEFORE the event (deaka'd names)"""
    out = []
    hands, public, racc = [Counter() for _ in range(4)], Counter(), set()
    for ev in events:
        out.append(([Counter(h) for h in hands], Counter(public), set(racc)))
        ty = ev["type"]
        if ty == "start_kyoku":
            hands = [Counter(deaka(t) for t in h) for h in ev["tehais"]]
            public = Counter([deaka(ev["dora_marker"])]); racc = set()
        elif ty == "tsumo":
            hands[ev["actor"]][deaka(ev["pai"])] += 1
        elif ty == "dahai":
            hands[ev["actor"]][deaka(ev["pai"])] -= 1; public[deaka(ev["pai"])] += 1
        elif ty in ("chi", "pon", "daiminkan", "ankan", "kakan"):
            cons = ev["consumed"] if ty != "kakan" else [ev["pai"]]
            for t in cons:
                hands[ev["actor"]][deaka(t)] -= 1; public[deaka(t)] += 1
        elif ty == "dora":
            public[deaka(ev["dora_marker"])] += 1
        elif ty == "reach_accepted":
            racc.add(ev["actor"])
    return out


def _dump(events):
    return "\n".join(json.dumps(e) for e in events) + "\n"


def mutate(events, cls: str, rng, tracked=None):
    """one mutation of class `cls` applied to a copy of `events` -> log text, or None when this log offers no place for it.
    tracked: track(events), when the caller already has it"""
    ev = [dict(e) for e in events]
    track_ = (lambda _: tracked) if tracked is not None else track
    idx = lambda pred: [i for i, e in enumerate(ev) if pred(e)]
    pick = lambda xs: xs[int(rng.integers(len(xs)))] if xs else None
    if cls == "dahai_not_held":
        st = track_(ev)
        cands = [(i, t) for i in idx(lambda e: e["type"] == "dahai") for t in TILES if st[i][0][ev[i]["actor"]][t] == 0]
        c = pick(cands)
        if c is None:
            return None
        ev[c[0]]["pai"] = c[1]; ev[c[0]]["tsumogiri"] = False
    elif cls == "dahai_illegal_held":
        st = track_(ev)
        cands = []
        for i in idx(lambda e: e["type"] == "dahai"):
            a = ev[i]["actor"]
            hand = st[i][0][a]
            if a in st[i][2]:  # after riichi only the drawn tile may go
                cands += [(i, t) for t, n in hand.items() if n > 0 and t != deaka(ev[i]["pai"])]
            elif i > 0 and ev[i - 1]["type"] == "chi" and ev[i - 1]["actor"] == a and hand[deaka(ev[i - 1]["pai"])] > 0:
                cands.append((i, deaka(ev[i - 1]["pai"])))  # kuikae: the tile just called
        c = pick(cands)
        if c is None:
            return None
        ev[c[0]]["pai"] = c[1]; ev[c[0]]["tsumogiri"] = False
    elif cls == "chi_non_kamicha":
        i = pick(idx(lambda e: e["type"] == "chi"))
        if i is None:
            return None
        ev[i]["target"] = (ev[i]["actor"] + int(rng.integers(1, 3))) % 4  # shimocha or toimen
    elif cls == "call_cannot":
        st = track_(ev)
        cands = [(i, s) for i in idx(lambda e: e["type"] == "dahai") for s in range(4)
                 if s != ev[i]["actor"] and st[i + 1][0][s][deaka(ev[i]["pai"])] < 2]
        c = pick(cands)
        if c is None:
            return None
        i, s = c
        d = ev[i]
        t = deaka(d["pai"])
        chi_seat = (d["actor"] + 1) % 4
        run = [f"{int(t[0]) - 2}{t[1]}", f"{int(t[0]) - 1}{t[1]}"] if t[0].isdigit() and int(t[0]) >= 3 else None
        if rng.integers(2) and run and min(st[i + 1][0][chi_seat][x] for x in run) == 0:  # the kamicha lacks a tile of the run
            ins = {"type": "chi", "actor": chi_seat, "target": d["actor"], "pai": d["pai"], "consumed": run}
        else:
            ins = {"type": "pon", "actor": s, "target": d["actor"], "pai": d["pai"], "consumed": [t, t]}
        ev.insert(i + 1, ins)
    elif cls == "riichi_not_tenpai":
        cands = idx(lambda e: e["type"] == "tsumo")
        i = pick([i for i in cands if i + 1 < len(ev) and ev[i + 1]["type"] == "dahai" and ev[i + 1]["actor"] == ev[i]["actor"]])
        if i is None:
            return None
        ev.insert(i + 1, {"type": "reach", "actor": ev[i]["actor"]})
    elif cls == "hora_non_winning":
        i = pick(idx(lambda e: e["type"] == "dahai"))
        if i is None:
            return None
        s = (ev[i]["actor"] + int(rng.integers(1, 4))) % 4
        ev.insert(i + 1, {"type": "hora", "actor": s, "target": ev[i]["actor"], "deltas": [0, 0, 0, 0], "ura_markers": []})
    elif cls == "deltas_lowered":
        i = pick(idx(lambda e: e["type"] == "hora" and e.get("deltas") is not None))
        if i is None:
            return None
        d = list(ev[i]["deltas"]); d[ev[i]["actor"]] = -int(rng.integers(1, 1000)); ev[i]["deltas"] = d
    elif cls == "hora_field_removed":
        i = pick(idx(lambda e: e["type"] == "hora"))
        if i is None:
            return None
        ev[i].pop("ura_markers" if rng.integers(2) else "deltas", None)
    elif cls == "tsumo_fifth":
        st = track_(ev)
        cands = [(i, t) for i in idx(lambda e: e["type"] == "tsumo") for t in TILES
                 if st[i][0][ev[i]["actor"]][t] + st[i][1][t] >= 4]
        c = pick(cands)
        if c is None:
            return None
        ev[c[0]]["pai"] = c[1]
    elif cls == "haipai_unknown":
        i = pick(idx(lambda e: e["type"] == "start_kyoku"))
        if i is None:
            return None
        th = [list(h) for h in ev[i]["tehais"]]
        th[int(rng.integers(4))][int(rng.integers(13))] = "?"
        ev[i]["tehais"] = th
    elif cls == "unparsable":
        i = int(rng.integers(len(ev)))
        text = _dump(ev).splitlines()
        text[i] = text[i][: int(rng.integers(1, max(2, len(text[i]) - 1)))]
        return "\n".join(text) + "\n"
    else:
        raise ValueError(cls)
    return _dump(ev)


def mutated_corpus(games, n_per_class: int, rng):
    """[(class, text)]: n_per_class mutations of every class, each over a randomly chosen game"""
    out, cache = [], {}
    for cls in CLASSES:
        made = tries = 0
        while made < n_per_class and tries < 50 * n_per_class:
            tries += 1
            g = int(rng.integers(len(games)))
            if g not in cache:
                cache[g] = track(games[g])
            t = mutate(games[g], cls, rng, cache[g])
            if t is not None:
                out.append((cls, t)); made += 1
    return out


def _random_word(rng):
    b = rng.integers(0, 256, size=8)
    b[0] = rng.integers(0, 20)  # mostly real event types, a few beyond them
    for k in (1, 3, 4, 5, 6):
        if rng.integers(4):
            b[k] = rng.integers(0, 41)  # tiles around the valid range (36 = 5sr, 37 = `?`)
    return int.from_bytes(bytes(int(x) for x in b), "little")


def malformed_batch(encoded, n, rng):
    """`n` hostile logs in validate_logs.pack() layout: event words of valid logs (encoded: validate_logs.EncodedLog list) with
    random words inserted or overwritten, random payload / hora bytes, or wholly random word sequences"""
    from mortal_b200.validate_logs import EncodedLog, pack

    out = []
    for i in range(n):
        e = encoded[int(rng.integers(len(encoded)))]
        hdr, ky, ho = e.hdr.copy(), e.kyoku.copy(), e.hora.copy()
        kind = int(rng.integers(4))
        if kind == 0:
            hdr = np.array([_random_word(rng) for _ in range(int(rng.integers(1, 200)))], dtype=np.uint64)
        elif kind == 1:
            for _ in range(int(rng.integers(1, 8))):
                j = int(rng.integers(len(hdr)))
                hdr[j] = _random_word(rng)
        elif kind == 2:
            for _ in range(int(rng.integers(1, 8))):
                j = int(rng.integers(len(hdr) + 1))
                hdr = np.insert(hdr, j, np.uint64(_random_word(rng)))
        else:
            if len(ky):
                ky[int(rng.integers(len(ky)))] = rng.integers(0, 2**63, size=ky.shape[1], dtype=np.uint64)
            if len(ho):
                ho[int(rng.integers(len(ho)))] = rng.integers(0, 2**63, size=ho.shape[1], dtype=np.uint64)
            hdr[int(rng.integers(len(hdr)))] = _random_word(rng)
        # the payload cursors may run past the arrays: drop trailing payloads / entries now and then
        if rng.integers(3) == 0:
            ky = ky[: int(rng.integers(len(ky) + 1))]
            ho = ho[: int(rng.integers(len(ho) + 1))]
        out.append(EncodedLog(hdr, ky.reshape(-1, ky.shape[-1] if ky.ndim == 2 else 19), ho.reshape(-1, 2), [], []))
    return pack(out)
