"""Helpers of the single-viewpoint loader tests — TEST INFRASTRUCTURE: the log the mjai protocol shows one seat and the scan
k_replay_viewpoints makes, restated over mjai events. The host build of the scan is emul_lib.EmulReplay.viewpoints()."""
from __future__ import annotations


def named(events):
    """the log with four distinct player names (`<name>.<seat>`), so that player_names selects exactly one seat"""
    first = dict(events[0])
    names = list(first.get("names", ["", "", "", ""]))
    first["names"] = [f"{nm}.{s}" for s, nm in enumerate(names)]
    return [first] + list(events[1:])


def viewpoint(events, p):
    """the log as seat p's mjai client receives it: the other seats' haipai are 13 x "?" and their draws "pai": "?"; with
    named()'s distinct names"""
    out = []
    for ev in named(events):
        if ev["type"] == "start_kyoku":
            ev = {**ev, "tehais": [list(h) if s == p else ["?"] * 13 for s, h in enumerate(ev["tehais"])]}
        elif ev["type"] == "tsumo" and ev["actor"] != p:
            ev = {**ev, "pai": "?"}
        out.append(ev)
    return out


def hidden_seats(events):
    """the mask k_replay_viewpoints computes: bit s when a haipai tile of seat s or a tsumo of seat s is "?" """
    m = 0
    for ev in events:
        if ev["type"] == "start_kyoku":
            for s, h in enumerate(ev["tehais"]):
                if "?" in h:
                    m |= 1 << s
        elif ev["type"] == "tsumo" and ev["pai"] == "?":
            m |= 1 << ev["actor"]
    return m
