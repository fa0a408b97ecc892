"""Pins the oracle's algo layer to the reference's own known-answer tests.

Transcribed from Mortal's libriichi/src: algo/shanten.rs:157-202, algo/agari.rs:919-1380,
algo/point.rs:120-154, rankings.rs:29-66.
"""
import numpy as np
import pytest

import oracle_lib as O
from oracle_lib import hand, tid


def sh(s, n):
    return int(O.shanten(hand(s), n)[0])


def test_shanten_3n_plus_1():  # shanten.rs:157-177
    assert sh("1111m 333p 222s 444z", 4) == 1
    assert sh("147m 258p 369s 1234z", 4) == 6
    assert sh("468m 33346p 7s", 3) == 2
    assert sh("147m 258p 3s", 2) == 4
    assert sh("4455s", 1) == 0
    assert sh("7z", 0) == 0
    assert sh("15559m 19p 19s 1234z", 4) == 3
    assert sh("9999m 6677p 88s 355z", 4) == 2
    assert sh("19m 19p 159s 123456z", 4) == 1


def test_shanten_3n_plus_2():  # shanten.rs:179-201
    assert sh("2344456m 14p 127s 2z 7p", 4) == 3
    assert sh("2344456m 14p 127s 2z 5p", 4) == 2
    assert sh("344455667p 1139s 9m", 4) == 2
    assert sh("344455667p 1139s 9p", 4) == 1
    assert sh("122334m 678p 37s 22z 5s", 4) == 0
    assert sh("122334m 678p 12s 22z 4s", 4) == 0
    assert sh("12223456m 78889p 2m", 4) == -1
    assert sh("34778p", 1) == 0
    assert sh("34s", 0) == 0
    assert sh("55m", 0) == -1


def test_ankan_after_riichi():  # agari.rs:919-957
    def one(tehai_str, tile, len_div3, strict, expected):
        t = hand(tehai_str)
        t[tid(tile)] += 1
        r = O.lib().orc_check_ankan_after_riichi(t.ctypes.data, len_div3, tid(tile), int(strict))
        assert r == int(expected), (tehai_str, tile, strict)

    one("12345m 567s 11222z", "S", 4, True, True)
    one("12345m 444567s 11z", "4s", 4, True, True)
    one("22m 11112356p 444s", "4s", 4, True, True)
    one("123456m 4445s 111z", "4s", 4, True, False)
    one("123456m 4445s 111z", "4s", 4, False, False)
    one("1113444p 222z", "1p", 3, True, False)
    one("1113444p 222z", "1p", 3, False, True)
    one("1113444p 222z", "4p", 3, True, False)
    one("1113444p 222z", "S", 3, True, True)
    one("23m 999p 33345666s", "3s", 4, True, False)
    one("23m 999p 33345666s", "6s", 4, True, False)
    one("23m 999p 33345666s", "6s", 4, False, True)
    one("23m 999p 33345666s", "9p", 4, True, True)
    one("1113445678999m", "1m", 4, True, True)
    one("1113445678999m", "9m", 4, True, False)


def yakus(tehai, **kw):
    r = O.agari(O.agari_query(tehai, **kw), 0)[0]
    if r["kind"] == 0:
        return None
    if r["kind"] == 2:
        return ("yakuman", int(r["yakuman"]))
    return (int(r["fu"]), int(r["han"]))


# agari.rs:959-1380 — (tehai, kwargs, expected); expected (fu, han), ("yakuman", n), None, or ("han", n)
AGARI_KATS = [
    ("2234455m 234p 234s 3m", dict(bakaze="E", jikaze="S", winning_tile="3m", is_ron=True), (40, 4)),
    ("2255m 445p 667788s 5p", dict(bakaze="E", jikaze="S", winning_tile="5p", is_ron=True), (25, 3)),
    ("22334m 33p 4m", dict(chis=["2s", "2s"], bakaze="E", jikaze="S", winning_tile="4m", is_ron=True), (30, 1)),
    ("223344p 667788s 3m 3m", dict(bakaze="S", jikaze="N", winning_tile="3m", is_ron=False), (30, 4)),
    ("234678m 1123488p 8p", dict(bakaze="E", jikaze="E", winning_tile="8p", is_ron=True), None),
    ("223344999m 1188p 8p", dict(bakaze="E", jikaze="E", winning_tile="8p", is_ron=True), (40, 1)),
    ("223344m 1188p 8p", dict(ankans=["9m"], bakaze="E", jikaze="E", winning_tile="8p", is_ron=True), (70, 1)),
    ("55566677m 11p 7m", dict(ankans=["9s"], bakaze="E", jikaze="E", winning_tile="7m", is_ron=False), ("yakuman", 1)),
    ("55566677m 11p 7m", dict(ankans=["9s"], bakaze="E", jikaze="E", winning_tile="7m", is_ron=True), (80, 4)),
    ("666677778888m 99p", dict(bakaze="E", jikaze="E", winning_tile="8m", is_ron=True), (30, 4)),
    ("666677778888m 99p", dict(bakaze="E", jikaze="E", winning_tile="7m", is_ron=True), (40, 3)),
    ("12345678m 11p 9m", dict(ankans=["9p"], bakaze="E", jikaze="E", winning_tile="9m", is_ron=True), (70, 2)),
    ("12345678m 11p 9m", dict(pons=["9p"], bakaze="E", jikaze="E", winning_tile="9m", is_ron=True), (30, 1)),
    ("111222333m 67p 88s 8p", dict(bakaze="E", jikaze="E", winning_tile="8p", is_ron=False), (40, 2)),
    ("1112223334447z 7z", dict(bakaze="E", jikaze="E", winning_tile="C", is_ron=True), ("yakuman", 3)),
    ("1m 789p 789s 1m", dict(chis=["7m", "1s"], bakaze="E", jikaze="E", winning_tile="1m", is_ron=False), (30, 3)),
    ("111444m 45556s 22z 5s", dict(bakaze="S", jikaze="S", winning_tile="5s", is_ron=True), (60, 2)),
    ("999s 1777z 1z", dict(chis=["1p"], pons=["N"], bakaze="S", jikaze="S", winning_tile="E", is_ron=True), (50, 2)),
    ("1119m 9m", dict(pons=["S", "C"], ankans=["N"], bakaze="S", jikaze="N", winning_tile="9m", is_ron=True), ("han", 9)),
    ("1233334567888m 9m", dict(bakaze="E", jikaze="E", winning_tile="9m", is_ron=True), ("han", 8)),
    ("2344445666678p 5p", dict(bakaze="E", jikaze="E", winning_tile="5p", is_ron=True), ("han", 7)),
    ("2223445566s 1s", dict(chis=["7s"], bakaze="E", jikaze="E", winning_tile="1s", is_ron=True), ("han", 6)),
    ("1123444m 111p 111s 1m", dict(bakaze="E", jikaze="E", winning_tile="1m", is_ron=True), (60, 2)),
    ("111s 2225556677z 7z", dict(bakaze="S", jikaze="S", winning_tile="C", is_ron=True), ("han", 15)),
]


@pytest.mark.parametrize("tehai,kw,expected", AGARI_KATS)
def test_agari_kats(tehai, kw, expected):
    got = yakus(tehai, **kw)
    if isinstance(expected, tuple) and expected[0] == "han":
        assert got is not None and got[0] != "yakuman" and got[1] == expected[1]
    else:
        assert got == expected


def test_agari_points_and_fu_fallback():
    # agari.rs:977-1000: riichi + menzen tsumo on a yaku-less hand -> oya 7700 / 2600 all
    q = O.agari_query("12334m 345p 22s 777z 2m", bakaze="E", jikaze="E", winning_tile="3m", is_ron=False,
                      additional_hans=2, doras=0, is_oya=True)
    r = O.agari(q, 1)[0]
    assert (r["ron"], r["tsumo_ko"], r["tsumo_oya"]) == (7700, 2600, 0)
    # agari.rs:1014-1016: chiitoi 25fu 3han ko ron = 3200
    q = O.agari_query("2255m 445p 667788s 5p", bakaze="E", jikaze="S", winning_tile="5p", is_ron=True)
    assert O.agari(q, 0)[0]["ron"] == 3200
    # agari.rs:1300-1311: fu of the 9-han hand via calc_fu(false) == 70 -> agari() with 1 situational han, no yaku
    # path exercised through a yaku-less open hand: 234m chi, 567p pon-less... use additional_hans fallback
    q = O.agari_query("234678m 1123488p 8p", bakaze="E", jikaze="E", winning_tile="8p", is_ron=True,
                      additional_hans=1, doras=0)
    r = O.agari(q, 1)[0]
    # 20 + menzen ron 10 + 888p (minkou from ron, non-yaochuu 2)... winning tile fits shuntsu? no shuntsu with 8p
    assert r["kind"] == 1 and r["han"] == 1 and r["fu"] in (40,)


def test_point_table_matches_formula():  # point.rs:120-154
    for fu in list(range(20, 111, 10)) + [25]:
        for han in range(1, 15):
            if han == 1 and fu < 30:
                continue
            if han >= 13:
                base = 8000
            elif han >= 11:
                base = 6000
            elif han >= 8:
                base = 4000
            elif han >= 6:
                base = 3000
            elif han >= 5:
                base = 2000
            else:
                base = min(fu * 2 ** (2 + han), 2000)
            gp = lambda m: (base * m + 99) // 100 * 100
            out = (O.C.c_int32 * 3)()
            assert O.lib().orc_point(0, fu, han, out) == 0, (fu, han, O.err())
            assert (out[1], out[2], out[0]) == (gp(1), gp(2), gp(4)), (fu, han)
            assert O.lib().orc_point(1, fu, han, out) == 0
            assert (out[1], out[0]) == (gp(2), gp(6)), (fu, han)


def test_point_impossible_combination():  # point.rs:46,81 panics
    out = (O.C.c_int32 * 3)()
    assert O.lib().orc_point(0, 20, 1, out) != 0
    assert O.lib().orc_point(0, 120, 2, out) != 0
    assert O.lib().orc_point(0, 0, 5, out) == 0 and out[0] == 8000


def test_rankings():  # rankings.rs:29-66
    def rk(scores):
        s = np.array(scores, dtype=np.int32)
        pbr = np.zeros(4, dtype=np.uint8)
        rbp = np.zeros(4, dtype=np.uint8)
        O.lib().orc_rankings(s.ctypes.data, pbr.ctypes.data, rbp.ctypes.data)
        return list(pbr), list(rbp)

    assert rk([25000, 25000, 30000, 20000]) == ([2, 0, 1, 3], [1, 2, 0, 3])
    assert rk([25000, 25000, 25000, 25000]) == ([0, 1, 2, 3], [0, 1, 2, 3])
    assert rk([18000, 32000, 32000, 18000]) == ([1, 2, 0, 3], [2, 0, 1, 3])
    assert rk([32000, 18000, 18000, 32000]) == ([0, 3, 1, 2], [0, 2, 3, 1])
    assert rk([0, 100000, 0, 0]) == ([1, 0, 2, 3], [1, 0, 2, 3])


def test_agari_table_shape():  # agari.rs:22-51; SURVEY appendix A
    t14 = np.zeros(14, dtype=np.uint8)
    divs = np.zeros(4, dtype=np.uint32)
    key = O.lib().orc_agari_key(hand("2234455m 234p 234s 3m").ctypes.data, t14.ctypes.data)
    n = O.lib().orc_agari_lookup(key, divs.ctypes.data)
    assert n == 2 and all((int(d) >> 30) & 1 for d in divs[:n])  # both ipeikou
    key = O.lib().orc_agari_key(hand("19m 19p 19s 12345677z").ctypes.data, t14.ctypes.data)
    assert O.lib().orc_agari_lookup(key, divs.ctypes.data) == -1  # kokushi handled before lookup
