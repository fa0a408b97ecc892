"""k_stat_logs's logic (csrc/mjx_stat.cuh, host build) against Stat.from_game: per log and per seat mask, all 44 counters equal
the sum of from_game over the selected seats; the status is non-zero exactly where the host must decide; the reference report's
text for non-finite rates."""
import itertools
import json
import os

import numpy as np
import pytest

import log_mutations as LM
import stat_lib as S
from mortal_b200 import stat
from test_emul_vs_oracle import _selfplay_logs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASKS = list(range(16))


def _check(games, masks=MASKS):
    """every log under every mask: counters equal the host sum, status 0 (or the host raises and the status is non-zero)"""
    a = S.encode(games)
    for m in masks:
        out, status = S.run_emul(a, np.full(len(games), m))
        for i, ev in enumerate(games):
            want = S.host_row(ev, m)
            if want is None:
                assert status[i] != 0, (i, m)
                assert not out[i].any()
            else:
                assert status[i] == 0, (i, m, status[i])
                assert np.array_equal(out[i], want), (i, m, dict(zip(S.NAMES, out[i] - want)))


def test_counter_names_are_the_stat_counters():
    assert set(S.NAMES) == set(stat.COUNTERS) and len(S.NAMES) == len(stat.COUNTERS) == 44


def test_golden_game():
    with open(os.path.join(ROOT, "tests", "golden", "golden_game.jsonl")) as f:
        events = [json.loads(ln) for ln in f if ln.strip()]
    _check([events])


@pytest.fixture(scope="module")
def games():
    return _selfplay_logs(48, 1, 731000) + _selfplay_logs(24, 0, 732000)


def test_selfplay_logs(games):
    assert len(games) >= 64
    _check(games, masks=[1, 2, 4, 8, 15, 5])


def test_mutation_corpus(games):
    corpus = LM.mutated_corpus(games, 6, np.random.default_rng(11))
    assert {c for c, _ in corpus} == set(LM.CLASSES)
    parsed = []
    for _, text in corpus:
        try:
            parsed.append([json.loads(ln) for ln in text.splitlines() if ln.strip()])
        except ValueError:  # `unparsable`: the host raises, the decoder declines; nothing reaches the kernel
            continue
    assert len(parsed) >= 6 * (len(LM.CLASSES) - 1)
    _check(parsed, masks=[1, 2, 4, 8, 15])


# ---- hand-built logs --------------------------------------------------------------------------------------------------------
def _sk(oya=0, scores=(25000, 25000, 25000, 25000)):
    return {"type": "start_kyoku", "bakaze": "E", "dora_marker": "1m", "kyoku": oya + 1, "honba": 0, "kyotaku": 0, "oya": oya,
            "scores": list(scores), "tehais": [["1m"] * 13] * 4}


def _game(*kyoku, names=("a", "b", "c", "d")):
    return [{"type": "start_game", "names": list(names)}] + [e for k in kyoku for e in k] + [{"type": "end_game"}]


def _dahai(a):
    return {"type": "dahai", "actor": a, "pai": "1m", "tsumogiri": False}


def _reach(a):
    return [{"type": "reach", "actor": a}, _dahai(a), {"type": "reach_accepted", "actor": a}]


def _hora(a, t, deltas):
    return {"type": "hora", "actor": a, "target": t, "deltas": list(deltas)}


def _ryu(deltas):
    return {"type": "ryukyoku", "deltas": list(deltas)}


END = {"type": "end_kyoku"}
CHI = {"type": "chi", "actor": 1, "target": 0, "pai": "3m", "consumed": ["1m", "2m"]}
PON = {"type": "pon", "actor": 1, "target": 2, "pai": "5p", "consumed": ["5p", "5p"]}
DMK = {"type": "daiminkan", "actor": 2, "target": 3, "pai": "E", "consumed": ["E", "E", "E"]}
ANKAN = {"type": "ankan", "actor": 3, "consumed": ["C", "C", "C", "C"]}

EDGE = {
    "no start_kyoku": _game(),
    "four equal final scores": _game([_sk(), _dahai(0), _ryu([0, 0, 0, 0]), END]),
    "sum under 100000, tie at the top": _game([_sk(2, (30000, 30000, 20000, 19000)), _dahai(2), _ryu([0, 0, 0, 0]), END]),
    "dealer ron at 48000": _game([_sk(1), _dahai(0), _hora(1, 0, [-48000, 48000, 0, 0]), END]),
    "dealer ron at 47999": _game([_sk(1), _dahai(0), _hora(1, 0, [-47999, 47999, 0, 0]), END]),
    "non-dealer ron at 32000": _game([_sk(0), _dahai(3), _hora(2, 3, [0, 0, 32000, -32000]), END]),
    "non-dealer ron at 31999": _game([_sk(0), _dahai(3), _hora(2, 3, [0, 0, 31999, -31999]), END]),
    "riichi yakuman less the stick": _game([_sk(1), *_reach(1), _dahai(0), _hora(1, 0, [-48000, 49000, 0, 0]), END]),
    "ryukyoku delta 8000": _game([_sk(), _dahai(0), _ryu([8000, -4000, -2000, -2000]), END]),
    "ryukyoku delta 7999": _game([_sk(), _dahai(0), _ryu([7999, -4000, -2000, -1999]), END]),
    "double ron": _game([_sk(3), _dahai(0), _hora(1, 0, [-8000, 8000, 0, 0]), _hora(3, 0, [-12000, 0, 0, 12000]), END]),
    "riichi not accepted, then deal-in": _game([_sk(), _dahai(1), {"type": "reach", "actor": 2}, _dahai(2),
                                                _hora(3, 2, [0, 0, -5200, 5200]), END]),
    "others' riichi before and after": _game([_sk(), *_reach(0), _dahai(1), *_reach(1), _dahai(2), *_reach(2), *_reach(3),
                                              _ryu([-1500, -1500, -1500, 4500]), END]),
    "ankan beside chi, pon, daiminkan": _game([_sk(), _dahai(0), CHI, _dahai(1), PON, _dahai(1), DMK, _dahai(2), ANKAN,
                                               _dahai(3), _hora(1, 3, [0, 3900, 0, -3900]), END,
                                               _sk(1), ANKAN, _dahai(3), CHI, _dahai(1), _ryu([-1000, 3000, -1000, -1000]), END]),
    "duplicate names": _game([_sk(), *_reach(2), _dahai(3), _hora(2, 3, [0, 0, 9000, -8000]), END], names=("x", "y", "x", "z")),
    "tobi and a negative sum": _game([_sk(0, (1000, 20000, 30000, 40000)), _dahai(0), _hora(1, 0, [-18000, 18000, 0, 0]), END]),
    "scores past int32 when summed": _game([_sk(0, (2147483647, 2147483647, -2147483648, 5)), _dahai(0),
                                            _ryu([2147483647, 2147483647, 0, 0]), END]),
}


@pytest.mark.parametrize("name", list(EDGE))
def test_edge_cases(name):
    _check([EDGE[name]])


def test_thresholds_are_inclusive():
    k = {c: S.NAMES.index(c) for c in ("yakuman", "nagashi_mangan", "riichi_agari_point")}
    got = lambda name, m: S.run_emul(S.encode([EDGE[name]]), [m])[0][0]
    assert got("dealer ron at 48000", 2)[k["yakuman"]] == 1 and got("dealer ron at 47999", 2)[k["yakuman"]] == 0
    assert got("non-dealer ron at 32000", 4)[k["yakuman"]] == 1 and got("non-dealer ron at 31999", 4)[k["yakuman"]] == 0
    assert got("riichi yakuman less the stick", 2)[k["riichi_agari_point"]] == 48000
    assert got("ryukyoku delta 8000", 1)[k["nagashi_mangan"]] == 1 and got("ryukyoku delta 7999", 1)[k["nagashi_mangan"]] == 0


def test_duplicate_names_select_two_seats():
    ev = EDGE["duplicate names"]
    assert S.seat_mask(ev, "x") == 0b101
    out, status = S.run_emul(S.encode([ev]), [0b101])
    assert status[0] == 0 and out[0][S.NAMES.index("game")] == 2


# ---- the status ----------------------------------------------------------------------------------------------------------------
def _no_deltas(how, ty):
    ev = _game([_sk(), _dahai(0), _hora(1, 0, [-1000, 1000, 0, 0]) if ty == "hora" else _ryu([0, 0, 0, 0]), END])
    if how == "missing":
        del ev[3]["deltas"]
    else:
        ev[3]["deltas"] = None
    return ev


@pytest.mark.parametrize("how,ty", list(itertools.product(("missing", "null"), ("hora", "ryukyoku"))))
def test_status_for_unusable_deltas(how, ty):
    ev = _no_deltas(how, ty)
    a = S.encode([ev])
    for m in MASKS:
        out, status = S.run_emul(a, [m])
        want = S.host_row(ev, m)
        if m:
            assert want is None and status[0] == 2 and not out[0].any(), m
        else:  # no selected seat: the host reads nothing but the first event, and neither does the kernel
            assert want is not None and status[0] == 0 and not out[0].any(), m


def test_status_when_the_first_event_is_not_start_game():
    ev = EDGE["four equal final scores"][1:]
    for m in MASKS:
        out, status = S.run_emul(S.encode([ev]), [m])
        assert status[0] == 1 and not out[0].any()
    empty = S.encode([EDGE["no start_kyoku"], []])
    out, status = S.run_emul(empty, [15, 15])
    assert list(status) == [0, 1]


def test_status_is_zero_on_every_accepted_log(games):
    a = S.encode(games[:16])
    for m in MASKS:
        assert not S.run_emul(a, np.full(16, m))[1].any()


def test_hostile_arrays_are_bounded():
    """offsets and counts outside the arrays: CAPACITY, nothing read out of range (ASan: tests/sanitized_stat_run.py)"""
    base = S.encode([EDGE["double ron"], EDGE["ankan beside chi, pon, daiminkan"]])
    n_hdr, n_ky = len(base["hdr"]), len(base["kyoku"])
    cases = [dict(ev_off=[-1, 0]), dict(ev_off=[0, n_hdr]), dict(ev_cnt=[n_hdr + 1, 1]), dict(ev_cnt=[-3, 0]),
             dict(ky_off=[-1, 0]), dict(ky_off=[0, n_ky // 19])]
    for c in cases:
        a = {k: (np.array(c[k], dtype=np.int32) if k in c else v) for k, v in base.items()}
        out, status = S.run_emul(a, [15, 15])
        for i in range(2):
            assert status[i] in (0, 1, 3), (c, status)
            if status[i]:
                assert not out[i].any()
        assert 3 in status, c
    out, status = S.run_emul(base, [15, 15], n_hdr=n_hdr - 1, n_kyoku_words=n_ky)
    assert list(status) == [0, 3]
    out, status = S.run_emul(base, [15, 15], n_hdr=n_hdr, n_kyoku_words=n_ky - 19)
    assert list(status) == [0, 3]


def test_line_deltas_reader():
    cases = {b'{"type":"hora","actor":0,"target":1,"deltas":[-1,2,3,-2147483648]}': (True, [-1, 2, 3, -2147483648]),
             b' { "deltas" :\t[ 0 , 8000,-4000, -4000 ] , "type" : "ryukyoku" } ': (True, [0, 8000, -4000, -4000]),
             b'{"type":"hora","meta":{"deltas":[1,1,1,1]},"actor":0,"target":1,"deltas":null}': (False, [0, 0, 0, 0]),
             b'{"type":"ryukyoku","x":"\\"deltas\\":[1,2,3,4]"}': (False, [0, 0, 0, 0])}
    for line, want in cases.items():
        assert S.line_deltas(line) == want, line


# ---- the reference report --------------------------------------------------------------------------------------------------------
_EMPTY = """Games            0
Rounds           0
Rounds as dealer 0

1st (rate)       0 (NaN)
2nd (rate)       0 (NaN)
3rd (rate)       0 (NaN)
4th (rate)       0 (NaN)
Tobi(rate)       0 (NaN)
Avg rank         NaN
Total rank pt    0
Avg rank pt      NaN
Total Δscore     {point}
Avg game Δscore  {avg}
Avg round Δscore {avg}

Win rate      NaN
Deal-in rate  NaN
Call rate     NaN
Riichi rate   NaN
Ryukyoku rate NaN

Avg winning Δscore               NaN
Avg winning Δscore as dealer     NaN
Avg winning Δscore as non-dealer NaN
Avg riichi winning Δscore        NaN
Avg open winning Δscore          NaN
Avg dama winning Δscore          NaN
Avg ryukyoku Δscore              NaN

Avg winning turn        NaN
Avg riichi winning turn NaN
Avg open winning turn   NaN
Avg dama winning turn   NaN

Avg deal-in turn                 NaN
Avg deal-in Δscore               NaN
Avg deal-in Δscore to dealer     NaN
Avg deal-in Δscore to non-dealer NaN

Chasing riichi rate       NaN
Riichi chased rate        NaN
Winning rate after riichi NaN
Deal-in rate after riichi NaN
Avg riichi turn           NaN
Avg riichi Δscore         NaN

Avg number of calls     NaN
Winning rate after call NaN
Deal-in rate after call NaN
Avg call Δscore         NaN

Dealer wins/all dealer rounds  NaN
Dealer wins/all wins           NaN
Deal-in to dealer/all deal-ins NaN

Yakuman (rate)        0 (NaN)
Nagashi mangan (rate) 0 (NaN)"""


def test_reference_text_of_zero_denominators():
    assert stat.Stat().reference_text() == _EMPTY.format(point=0, avg="NaN")
    assert stat.Stat(point=-5).reference_text() == _EMPTY.format(point=-5, avg="-inf")
    assert stat.Stat(point=7).reference_text() == _EMPTY.format(point=7, avg="inf")


def test_reference_text_of_finite_rates():
    st = stat.Stat(game=3, round=7, rank_1=1, rank_2=2, yakuman=1, point=-10)
    text = st.reference_text()
    assert "1st (rate)       1 (0.333333)\n2nd (rate)       2 (0.666667)\n" in text
    assert "Avg game Δscore  -3.333333\n" in text and "Avg rank pt      60.000000\n" in text
    assert text.endswith("Yakuman (rate)        1 (0.142857143)\nNagashi mangan (rate) 0 (0.000000000)")


def test_cli_usage_exits_2(capsys):
    assert stat.main([]) == 2 and stat.main(["a"]) == 2 and stat.main(["a", "b", "c"]) == 2
    assert "Usage" in capsys.readouterr().err


# ---- from_dir's plumbing: chunks and device choice --------------------------------------------------------------------------------
def test_chunks_are_bounded_by_files_and_bytes(tmp_path, monkeypatch):
    import gzip
    from concurrent.futures import ThreadPoolExecutor

    sizes = [5, 40, 1, 100, 7, 7, 7, 30, 2, 0, 64]
    paths = []
    for k, n in enumerate(sizes):
        p = tmp_path / (f"{k:02d}.json.gz" if k % 2 else f"{k:02d}.json")
        p.write_bytes(gzip.compress(b"x" * n) if k % 2 else b"x" * n)
        paths.append(str(p))
    bad = tmp_path / "bad.json.gz"
    bad.write_bytes(b"not gzip")
    paths.insert(4, str(bad))
    monkeypatch.setattr(stat, "CHUNK_BYTES", 48)
    monkeypatch.setattr(stat, "CHUNK_LOGS", 3)
    with ThreadPoolExecutor(2) as pool:
        chunks = list(stat._chunks(paths, pool, 3))
    assert [p for c, _ in chunks for p in c] == paths
    for c, blobs in chunks:
        assert len(c) == len(blobs) and 1 <= len(c) <= 3
        size = sum(len(b) for b in blobs if b is not None)
        assert size <= 48 or len(c) == 1, (c, size)
        for p, b in zip(c, blobs):
            assert (b is None) == (p == str(bad))
    assert sum(len(b) for _, bs in chunks for b in bs if b is not None) == sum(sizes)


def test_from_dir_runs_on_the_device_libmjx_is_initialised_on(monkeypatch):
    from mortal_b200 import _lib

    monkeypatch.setattr(_lib, "_INIT_DEVICE", 3)  # e.g. an arena or engine on cuda:3 in this process
    assert stat._stat_device() == 3
