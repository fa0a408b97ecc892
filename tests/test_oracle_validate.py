"""bin/validate_logs.rs process_path restated by the oracle (oracle/validate.cc): the reference's own log is valid, and hand-built
mutations of it fail the check or update the reference code names, at the line it names."""
import json
import os

import pytest

from validate_lib import V, emul_validate, oracle_validate

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_game.jsonl")


def _log():
    with open(GOLDEN) as f:
        return [json.loads(x) for x in f.read().splitlines()]


def _text(events):
    return "\n".join(json.dumps(e) for e in events) + "\n"


def _edit(line, **fields):
    def f(ev):
        ev[line - 1] = {**ev[line - 1], **fields}
    return f


def _drop(line, key):
    def f(ev):
        ev[line - 1] = {k: v for k, v in ev[line - 1].items() if k != key}
    return f


def _insert(after, *new):
    def f(ev):
        ev[after:after] = list(new)
    return f


# (mutation, expected verdict): lines refer to tests/golden/golden_game.jsonl (3: seat 0 draws 1s; 4: seat 0 discards W holding
# 1p 1p 1s 2p 3m 3p 4p 5m 5s 6m 6m 6s P W; 35: seat 2 pons E from seat 3; 79: seat 0 rons seat 2 after riichi; 142: seat 1 chis
# 2s with 3s 4s from seat 0)
CASES = {
    # validate_logs.rs:86-99
    "can_discard": (_edit(12, actor=1), V("CHECK", "can_discard", 12, 1)),
    "discard_candidates": (_edit(4, pai="9p", tsumogiri=False), V("CHECK", "discard_candidates", 4, 0)),
    # :100-139
    "chi_non_kamicha": (_edit(142, target=3), V("CHECK", "chi from non-kamicha", 142, 1)),
    "can_chi_low": (_insert(8, {"type": "chi", "actor": 3, "target": 2, "pai": "1s", "consumed": ["2s", "3s"]}),
                    V("CHECK", "can_chi_low", 9, 3)),
    "can_chi_mid": (_edit(142, consumed=["1s", "3s"]), V("CHECK", "can_chi_mid", 142, 1)),
    "can_chi_high": (_insert(4, {"type": "chi", "actor": 1, "target": 0, "pai": "W", "consumed": ["3m", "4m"]}),
                     V("CHECK", "can_chi_high", 5, 1)),
    # :140-153
    "can_pon": (_insert(4, {"type": "pon", "actor": 2, "target": 0, "pai": "W", "consumed": ["W", "W"]}), V("CHECK", "can_pon", 5, 2)),
    "can_daiminkan": (_insert(4, {"type": "daiminkan", "actor": 3, "target": 0, "pai": "W", "consumed": ["W", "W", "W"]}),
                      V("CHECK", "can_daiminkan", 5, 3)),
    # :154-181
    "can_ankan": (_insert(3, {"type": "ankan", "actor": 0, "consumed": ["6m", "6m", "6m", "6m"]}), V("CHECK", "can_ankan", 4, 0)),
    "can_kakan": (_insert(37, {"type": "kakan", "actor": 2, "pai": "E", "consumed": ["E", "E", "E"]}), V("CHECK", "can_kakan", 38, 2)),
    # :182-188
    "can_riichi": (_insert(3, {"type": "reach", "actor": 0}), V("CHECK", "can_riichi", 4, 0)),
    # :189-232
    "can_ron_agari": (_insert(4, {"type": "hora", "actor": 1, "target": 0, "deltas": [0, 0, 0, 0], "ura_markers": []}),
                      V("CHECK", "can_ron_agari", 5, 1)),
    "can_tsumo_agari": (_insert(3, {"type": "hora", "actor": 0, "target": 0, "deltas": [0, 0, 0, 0], "ura_markers": []}),
                        V("CHECK", "can_tsumo_agari", 4, 0)),
    "missing_ura": (_drop(79, "ura_markers"), V("CHECK", "missing ura_markers", 79, 0)),
    "missing_deltas": (_drop(79, "deltas"), V("CHECK", "missing deltas", 79, 0)),
    "deltas_below_points": (_edit(79, deltas=[100, 0, -100, 0]), V("CHECK", "deltas below points", 79, 0)),
    # update.rs errors, lowest seat first
    "unknown_tile": (lambda ev: ev.__setitem__(1, {**ev[1], "tehais": [ev[1]["tehais"][0], ["?"] + ev[1]["tehais"][1][1:]]
                                                   + ev[1]["tehais"][2:]}), V("UPDATE", "witness unknown tile", 2, 1)),
    "fifth_tile": (_edit(75, pai="4s"), V("UPDATE", "witness fifth tile", 75, 1)),
    "consume_from_void": (_edit(35, consumed=["1m", "1m"]), V("UPDATE", "consume from void", 35, 2)),
    # a low chi seat 1 may make (2s with 3s 4s) passes the check; consuming a 9s it does not hold fails its own update
    "consume_from_void_chi": (_edit(142, consumed=["9s", "8s"]), V("UPDATE", "consume from void", 142, 1)),
    "dora_overflow": (_insert(3, *[{"type": "dora", "dora_marker": t} for t in ("1m", "2m", "3m", "4m", "5m")]),
                      V("UPDATE", "dora indicator overflow", 8, 0)),
    # host-side parse
    "json": (lambda ev: ev.__setitem__(9, "{\"type\": \"dahai\""), V("PARSE", "json", 10)),
    "unknown_type": (_edit(10, type="discard"), V("PARSE", "unknown type", 10)),
    "unknown_tile_name": (_edit(10, pai="0m"), V("PARSE", "unknown tile", 10)),
    "actor_range": (_edit(10, actor=4), V("PARSE", "actor out of range", 10)),
    "consumed_length": (_edit(35, consumed=["E"]), V("PARSE", "consumed length", 35)),
    "missing_field": (_drop(10, "tsumogiri"), V("PARSE", "missing or invalid field", 10)),
}


def _mutated(name):
    ev = _log()
    CASES[name][0](ev)
    return "\n".join(e if isinstance(e, str) else json.dumps(e) for e in ev) + "\n"


def test_golden_log_is_valid():
    assert oracle_validate(_text(_log())) is None


@pytest.mark.parametrize("name", sorted(CASES))
def test_mutation_verdict(name):
    text = _mutated(name)
    assert oracle_validate(text) == CASES[name][1]


def test_emulated_kernel_agrees_on_the_golden_mutations():
    names = sorted(CASES)
    texts = [_text(_log())] + [_mutated(n) for n in names]
    assert emul_validate(texts) == [None] + [CASES[n][1] for n in names]
