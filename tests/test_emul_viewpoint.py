"""Single-viewpoint logs in the log replay (k_replay_viewpoints + the single-viewer record, host-emulated): a log that hides the other
seats' tiles, as the mjai protocol shows a game to one seat, replays for that seat to exactly the rows of the full log, and to the
oracle's restatement of dataset/gameplay.rs (one PlayerState, so it takes such logs as the reference does); full-information logs
replay bit for bit as without the scan; a job whose own tiles are hidden fails with code 13 and leaves the other jobs alone."""
import json
import os

import numpy as np
import pytest

import oracle_lib as O
import validate_lib as VL
from emul_lib import EmulReplay
from viewpoint_lib import hidden_seats, named, viewpoint

HERE = os.path.dirname(os.path.abspath(__file__))
ERR_HIDDEN_OWN_TILE = 13


def _golden():
    with open(os.path.join(HERE, "golden", "golden_game.jsonl")) as f:
        return [{k: v for k, v in json.loads(ln).items() if k != "meta"} for ln in f if ln.strip()]


@pytest.fixture(scope="module")
def logs():
    """the golden game and self-play logs of both test-policy kinds"""
    return [_golden()] + VL.emul_games(4, 1, seed0=7300) + VL.emul_games(4, 0, seed0=7400)


def _replay(games, players, *, view, obs=None, kan=True):
    """replay the jobs in one emulated env -> (per-job rows, per-job error codes, the scan's per-job result or None);
    obs = (version, single-player block) encodes every step's observations"""
    from mortal_b200 import dataset_codec as DC

    jobs = DC.build_jobs(games, players)
    rep = EmulReplay(jobs, always_include_kan_select=kan)
    scan = rep.viewpoints() if view else None
    per = [dict(actions=[], masks=[], meta=[], obs=[]) for _ in range(rep.n_tables)]
    for _ in range(10000):
        rep.replay_step()
        if rep.num_rows():
            rt, _, m = rep.rows()
            lab, meta = rep.row_labels()
            o = rep.encode_obs(sp=obs[1], version=obs[0]) if obs else None
            for r in range(len(rt)):
                j = per[rt[r]]
                j["actions"].append(int(lab[r])); j["masks"].append(m[r]); j["meta"].append(meta[r].copy())
                if obs:
                    j["obs"].append(o[r])
        if rep.live == 0:
            break
    assert rep.live == 0
    errs = rep.errs()
    rep.close()
    return per, errs, scan


def _same_rows(a, b, obs=False):
    assert a["actions"] == b["actions"]
    assert np.array_equal(np.array(a["masks"]), np.array(b["masks"])) and np.array_equal(np.array(a["meta"]), np.array(b["meta"]))
    if obs:
        ga, gb = np.array(a["obs"]), np.array(b["obs"])
        assert ga.shape == gb.shape and ga.tobytes() == gb.tobytes()  # bit-identical


def test_viewpoint_logs_match_the_oracle_and_the_full_log(logs):
    """for every seat p, viewpoint(L, p) replayed with the scan gives p's rows of the full log L and of the oracle's loader"""
    games = [viewpoint(L, p) for L in logs for p in range(4)]
    players = [[p] for _ in logs for p in range(4)]
    got, errs, scan = _replay(games, players, view=True)
    full, ferrs, _ = _replay(logs, [[0, 1, 2, 3]] * len(logs), view=False)
    assert not errs.any() and not ferrs.any()
    assert scan.tolist() == [0xF & ~(1 << p) for _ in logs for p in range(4)]
    assert scan.tolist() == [hidden_seats(g) for g in games]
    moves = 0
    for j, (g, pl) in enumerate(zip(games, players)):
        p = pl[0]
        _same_rows(got[j], full[j])  # job j of the full replay is log j // 4, player j % 4
        ref = O.gameplay_load(g, p, with_obs=False, sp_mode=0)
        meta = np.array(got[j]["meta"])
        assert got[j]["actions"] == ref["actions"].tolist(), j
        assert (np.array(got[j]["masks"]) == ref["masks"]).all(), j
        assert (meta[:, 0] == ref["at_kyoku"]).all() and (meta[:, 1] == ref["at_turns"]).all(), j
        assert (meta[:, 2].astype(np.int8) == ref["shantens"]).all() and (meta[:, 3].astype(bool) == ref["apply_gamma"]).all(), j
        moves += len(got[j]["actions"])
    assert moves > 3000


@pytest.mark.parametrize("version,sp", [(4, True), (3, False), (1, False)])
def test_viewpoint_observations_are_bit_identical_to_the_full_log(logs, version, sp):
    sel = logs[:5] if sp else logs
    games = [viewpoint(L, p) for L in sel for p in range(4)]
    got, errs, _ = _replay(games, [[p] for _ in sel for p in range(4)], view=True, obs=(version, sp))
    full, ferrs, _ = _replay(sel, [[0, 1, 2, 3]] * len(sel), view=False, obs=(version, sp))
    assert not errs.any() and not ferrs.any()
    for j in range(len(games)):
        _same_rows(got[j], full[j], obs=True)
    if sp:  # the single-player block (rows 889-1011 of v4) is really computed
        assert any(np.array(j["obs"])[:, 889:].any() for j in got)


def test_viewpoint_without_kan_select_rows(logs):
    games = [viewpoint(L, p) for L in logs[:4] for p in range(4)]
    got, errs, _ = _replay(games, [[p] for _ in logs[:4] for p in range(4)], view=True, kan=False)
    full, _, _ = _replay(logs[:4], [[0, 1, 2, 3]] * 4, view=False, kan=False)
    assert not errs.any()
    for j in range(len(games)):
        _same_rows(got[j], full[j])


def test_full_information_logs_replay_unchanged(logs):
    """the scan finds nothing on a full-information log and writes nothing: rows and observations as without it"""
    games = [named(L) for L in logs]
    a, ea, scan = _replay(games, [[0, 1, 2, 3]] * len(games), view=True, obs=(4, False))
    b, eb, _ = _replay(games, [[0, 1, 2, 3]] * len(games), view=False, obs=(4, False))
    assert not scan.any() and not ea.any() and not eb.any()
    for x, y in zip(a, b):
        _same_rows(x, y, obs=True)


def test_hidden_own_tiles_fail_with_code_13(logs):
    """in one env, the jobs whose own seat is hidden fail with code 13 at their first step; the other jobs' rows are unaffected"""
    L, M = logs[1], logs[5]
    games = [viewpoint(L, 1), viewpoint(L, 1), M, viewpoint(M, 3), viewpoint(M, 3)]
    players = [[1, 2], [0], [0, 2], [3], [0, 3]]
    got, errs, scan = _replay(games, players, view=True)
    assert errs.tolist() == [0, ERR_HIDDEN_OWN_TILE, ERR_HIDDEN_OWN_TILE, 0, 0, 0, ERR_HIDDEN_OWN_TILE, 0]
    assert scan.tolist() == [0xD, 0xD, 0xD, 0, 0, 0x7, 0x7, 0x7]
    for j in (1, 2, 6):
        assert got[j]["actions"] == []
    alone, _, _ = _replay([viewpoint(L, 1), M, viewpoint(M, 3)], [[1], [0, 2], [3]], view=True)
    for j, k in ((0, 0), (3, 1), (4, 2), (5, 3), (7, 3)):
        _same_rows(got[j], alone[k])


def _jobs(games, players):
    from mortal_b200 import dataset_codec as DC

    return DC.build_jobs(games, players)


def test_scan_edge_cases(logs):
    """short jobs, start_kyoku words without a payload left, and `?` outside the haipai and draws"""
    L = logs[2]
    ky = [i for i, ev in enumerate(L) if ev["type"] == "start_kyoku"]
    v = viewpoint(L, 0)
    # `?` in a dora marker and in consumed tiles does not hide a seat
    odd = [dict(ev) for ev in L]
    odd[ky[0]]["dora_marker"] = "?"
    k = next(i for i, ev in enumerate(odd) if ev["type"] in ("chi", "pon"))
    odd[k]["consumed"] = ["?", "?"]
    all_q = [{**ev, "tehais": [["?"] * 13] * 4} if ev["type"] == "start_kyoku" else ev for ev in viewpoint(L, 0)]
    games = [[], v[:1], v[:2], v[:3], v[ky[0]:ky[0] + 1], odd, all_q]
    a = _jobs(games, [[0]] * len(games))
    rep = EmulReplay(a)
    scan = rep.viewpoints()
    rep.close()
    assert scan.tolist() == [hidden_seats(g) for g in games] == [0, 0, 0xE, 0xE, 0xE, 0, 0xF]
    # a job with more start_kyoku words than payloads left is not marked (-1)
    short = dict(a, kyoku=a["kyoku"][: 19 * int(a["ky_off"][4])])
    rep = EmulReplay(short)
    scan = rep.viewpoints()
    rep.close()
    assert scan.tolist() == [0, 0, 0xE, 0xE, -1, -1, -1]
