"""The assertions of the reference's state tests (Mortal's libriichi/src/state/test.rs, line refs inline), written
against the libriichi.state.PlayerState surface so that the same bodies run on the oracle (tests/test_oracle_state.py keeps its
own copy), on the host-emulated product (tests/test_emul_state.py) and on the CUDA path (tests/test_gpu_state.py).
Inline mjai logs: tests/golden/state_test_logs.json (tools/extract_ref_fixtures.py)."""
import json
import os

import numpy as np

import oracle_lib as O

HERE = os.path.dirname(os.path.abspath(__file__))
with open(os.path.join(HERE, "golden", "state_test_logs.json")) as f:
    LOGS = json.load(f)
UNK13 = ["?"] * 13
tid = O.tid


def tiles_of(s):
    h = O.hand_with_aka(s)
    out = []
    for t in range(37):
        out += [O.TILE_NAMES[t]] * int(h[t])
    return out


def validate(ps):
    """test.rs:49-67 after every update"""
    v = ps.view()
    th = np.array(list(v.tehai), dtype=np.uint8)
    assert v.real_time_shanten == int(O.shanten(th, v.tehai_len_div3)[0])
    assert bool(v.is_menzen) == (v.n_chis == 0 and v.n_pons == 0 and v.n_minkans == 0)
    if ps.last_cans.can_act:
        for version in (1, 2, 3, 4):
            obs, mask = ps.encode_obs(version, False)
            assert obs.shape[1] == 34 and obs.min() >= 0.0 and obs.max() <= 1.0 and mask.shape == (46,)
            if ps.last_cans.can_kakan or ps.last_cans.can_ankan:
                ps.encode_obs(version, True)


def upd(ps, ev, check=True):
    cans = ps.update(ev if isinstance(ev, str) else json.dumps(ev))
    if check:
        validate(ps)
    return cans


def from_log(PS, pid, lines):
    ps = PS(pid)
    for ln in lines:
        upd(ps, ln)
    return ps


def start_kyoku(tehai0, dora, **kw):
    d = dict(type="start_kyoku", bakaze="E", kyoku=1, honba=0, kyotaku=0, oya=0, scores=[25000] * 4,
             dora_marker=dora, tehais=[tiles_of(tehai0), UNK13, UNK13, UNK13])
    d.update(kw)
    return d


def case_furiten(PS):  # test.rs:223-477
    ps = PS(0)
    upd(ps, start_kyoku("23406m 456789p 58s", "3p"))
    upd(ps, dict(type="tsumo", actor=0, pai="8s"))
    v = ps.view()
    assert v.shanten == 1 and not any(v.waits)
    upd(ps, dict(type="dahai", actor=0, pai="5s", tsumogiri=False))
    v = ps.view()
    assert v.shanten == 0 and v.waits[tid("1m")] and v.waits[tid("4m")] and v.waits[tid("7m")] and not v.at_furiten
    upd(ps, dict(type="tsumo", actor=1, pai="?"))
    cans = upd(ps, dict(type="dahai", actor=1, pai="1m", tsumogiri=False))
    assert not ps.view().at_furiten and cans.can_ron_agari
    upd(ps, dict(type="tsumo", actor=2, pai="?"))
    assert ps.view().at_furiten  # same-cycle furiten
    upd(ps, dict(type="dahai", actor=2, pai="1s", tsumogiri=True))
    upd(ps, dict(type="tsumo", actor=3, pai="?"))
    cans = upd(ps, dict(type="dahai", actor=3, pai="1m", tsumogiri=False))
    v = ps.view()
    assert v.shanten == 0 and v.at_furiten and not cans.can_ron_agari
    upd(ps, dict(type="tsumo", actor=0, pai="3s"))
    assert ps.view().at_furiten
    upd(ps, dict(type="dahai", actor=0, pai="3s", tsumogiri=True))
    assert not ps.view().at_furiten
    for actor, pai in ((1, "P"), (2, "C")):
        upd(ps, dict(type="tsumo", actor=actor, pai="?"))
        upd(ps, dict(type="dahai", actor=actor, pai=pai, tsumogiri=True))
    upd(ps, dict(type="tsumo", actor=3, pai="?"))
    cans = upd(ps, dict(type="dahai", actor=3, pai="1m", tsumogiri=False))
    assert not ps.view().at_furiten and cans.can_ron_agari
    assert ps.agari_points(True)["ron"] == 5800  # test.rs:337
    cans = upd(ps, dict(type="tsumo", actor=0, pai="N"))
    assert cans.can_riichi
    ps.validate_reaction(json.dumps(dict(type="reach", actor=0)))
    upd(ps, dict(type="reach", actor=0))
    upd(ps, dict(type="dahai", actor=0, pai="N", tsumogiri=True))
    upd(ps, dict(type="reach_accepted", actor=0))
    assert ps.self_riichi_accepted
    for actor in (1, 2, 3):
        upd(ps, dict(type="tsumo", actor=actor, pai="?"))
        upd(ps, dict(type="dahai", actor=actor, pai="N", tsumogiri=True))
    cans = upd(ps, dict(type="tsumo", actor=0, pai="7m"))
    v = ps.view()
    assert v.waits[tid("1m")] and v.waits[tid("4m")] and v.waits[tid("7m")] and not v.at_furiten and cans.can_tsumo_agari
    upd(ps, dict(type="dahai", actor=0, pai="7m", tsumogiri=True))
    assert ps.view().at_furiten  # furiten forever from now on
    upd(ps, dict(type="tsumo", actor=1, pai="?"))
    cans = upd(ps, dict(type="dahai", actor=1, pai="4m", tsumogiri=True))
    assert ps.view().at_furiten and not cans.can_ron_agari
    for actor in (2, 3):
        upd(ps, dict(type="tsumo", actor=actor, pai="?"))
        upd(ps, dict(type="dahai", actor=actor, pai="W", tsumogiri=True))
    assert ps.view().at_furiten
    cans = upd(ps, dict(type="tsumo", actor=0, pai="4m"))
    v = ps.view()
    assert v.waits[0] and v.waits[3] and v.waits[6] and v.at_furiten and cans.can_tsumo_agari
    assert ps.agari_points(False, ["3m"])["tsumo_ko"] == 6000  # test.rs:476


def case_dora_count_after_kan(PS):  # test.rs:479-579
    ps = PS(0)
    upd(ps, start_kyoku("1111s 123456p 112z", "N"))
    upd(ps, dict(type="tsumo", actor=0, pai="8s"))
    assert ps.view().doras_owned[0] == 2
    upd(ps, dict(type="ankan", actor=0, consumed=["1s"] * 4))
    upd(ps, dict(type="dora", dora_marker="9s"))
    upd(ps, dict(type="tsumo", actor=0, pai="5pr"))
    assert ps.view().doras_owned[0] == 7
    upd(ps, dict(type="dahai", actor=0, pai="E", tsumogiri=True))
    assert ps.view().doras_owned[0] == 6
    upd(ps, dict(type="tsumo", actor=1, pai="?"))
    upd(ps, dict(type="dahai", actor=1, pai="5p", tsumogiri=True))
    upd(ps, dict(type="pon", actor=0, target=1, pai="5p", consumed=["5pr", "5p"]))
    assert ps.view().doras_owned[0] == 6
    upd(ps, dict(type="dahai", actor=0, pai="E", tsumogiri=False))
    assert ps.view().doras_owned[0] == 5
    for actor in (1, 2):
        upd(ps, dict(type="tsumo", actor=actor, pai="?"))
        upd(ps, dict(type="dahai", actor=actor, pai="P", tsumogiri=True))
    upd(ps, dict(type="tsumo", actor=3, pai="?"))
    upd(ps, dict(type="ankan", actor=3, consumed=["1m"] * 4))
    upd(ps, dict(type="dora", dora_marker="4p"))
    assert ps.view().doras_owned[0] == 8


def case_rule_based_agari(PS):  # test.rs:581-799
    logs = LOGS["rule_based_agari_all_last_minogashi"]
    ps = from_log(PS, 1, logs[0])
    assert ps.last_cans.can_tsumo_agari and not ps.rule_based_agari()
    assert from_log(PS, 2, logs[1]).rule_based_agari()


def case_kakan_from_hand(PS):  # test.rs:828-911
    assert from_log(PS, 1, LOGS["kakan_from_hand"][0]).last_cans.can_tsumo_agari


def case_unconditional_tenpai(PS):  # test.rs:913-1224
    logs = LOGS["discard_candidates_with_unconditional_tenpai"]
    ps = from_log(PS, 1, logs[0])
    d = ps.discard_candidates(unconditional_tenpai=True)
    assert [O.TILE_NAMES[i] for i in range(34) if d[i]] == ["7p", "8p"]
    ps = from_log(PS, 1, logs[1])
    w = ps.waits
    assert [O.TILE_NAMES[i] for i in range(34) if w[i]] == ["5p", "8p"]
    assert not ps.discard_candidates(unconditional_tenpai=True).any()


def case_double_chankan_ron(PS):  # test.rs:1226-1391
    logs = LOGS["double_chankan_ron"]
    ps = from_log(PS, 2, logs[0])
    ps_kakan = ps.clone()
    cans = upd(ps_kakan, logs[1][0])
    assert cans.can_ron_agari and ps_kakan.agari_points(True)["ron"] == 1000
    assert not upd(ps, logs[2][0]).can_ron_agari


def case_chi_at_0_shanten(PS):  # test.rs:1393-1418
    logs = LOGS["chi_at_0_shanten"]
    ps = from_log(PS, 0, logs[0])
    v = ps.view()
    assert v.shanten == 0 and v.real_time_shanten == 0 and ps.last_cans.can_ron_agari and ps.last_cans.can_chi_high
    upd(ps, logs[1][0])
    v = ps.view()
    assert v.shanten == 0 and v.real_time_shanten == -1 and v.at_furiten and not v.has_next_shanten_discard


def case_getters_and_validation(PS):
    """state/getter.rs:6-156 and state/action.rs:93-227 on a small hand-made sequence"""
    import pytest

    ps = PS(2)
    sk = dict(type="start_kyoku", bakaze="S", kyoku=4, honba=2, kyotaku=1, oya=2, scores=[10000, 20000, 30000, 40000], dora_marker="1m",
              tehais=[UNK13, UNK13, tiles_of("123406m 4499p 11z 7s"), UNK13])
    cans = upd(ps, sk)
    assert not cans.can_act and ps.player_id == 2 and ps.kyoku == 3 and ps.honba == 2 and ps.kyotaku == 1 and ps.is_oya
    assert sum(ps.tehai) == 13 and ps.akas_in_hand == [True, False, False] and ps.at_turn == 0
    v = ps.view()
    assert list(v.scores) == [30000, 40000, 10000, 20000] and v.rank == 1 and v.is_all_last and O.TILE_NAMES[v.jikaze] == "E"
    cans = upd(ps, dict(type="tsumo", actor=2, pai="9p"))
    assert cans.can_discard and ps.last_self_tsumo() == "9p" and ps.at_turn == 1
    ps.validate_reaction(json.dumps(dict(type="dahai", actor=2, pai="9p", tsumogiri=True)))
    ps.validate_reaction(json.dumps(dict(type="dahai", actor=2, pai="5mr", tsumogiri=False)))
    for bad in (dict(type="dahai", actor=2, pai="2p", tsumogiri=False), dict(type="dahai", actor=2, pai="7s", tsumogiri=True),
                dict(type="dahai", actor=1, pai="9p", tsumogiri=True), dict(type="reach", actor=2) if not cans.can_riichi else dict(type="pon", actor=2, target=2, pai="1m", consumed=["1m", "1m"]),
                dict(type="hora", actor=2, target=2)):
        with pytest.raises(ValueError):
            ps.validate_reaction(json.dumps(bad))
    assert ps.decode_action(17) == {"type": "dahai", "actor": 2, "pai": "9p", "tsumogiri": True}
    assert ps.decode_action(34) == {"type": "dahai", "actor": 2, "pai": "5mr", "tsumogiri": False}
    upd(ps, dict(type="dahai", actor=2, pai="7s", tsumogiri=False))
    upd(ps, dict(type="tsumo", actor=3, pai="?"))
    cans = upd(ps, dict(type="dahai", actor=3, pai="9p", tsumogiri=False))
    assert cans.can_pon and cans.can_pass and cans.target_actor == 3 and ps.last_kawa_tile() == "9p"
    ps.validate_reaction(json.dumps(dict(type="pon", actor=2, target=3, pai="9p", consumed=["9p", "9p"])))
    ps.validate_reaction(json.dumps(dict(type="none")))
    assert ps.decode_action(41) == {"type": "pon", "actor": 2, "target": 3, "pai": "9p", "consumed": ["9p", "9p"]}
    assert ps.decode_action(45) == {"type": "none"}
    assert "shanten" in ps.brief_info()


ALL_CASES = [case_furiten, case_dora_count_after_kan, case_rule_based_agari, case_kakan_from_hand, case_unconditional_tenpai,
             case_double_chankan_ron, case_chi_at_0_shanten, case_getters_and_validation]
