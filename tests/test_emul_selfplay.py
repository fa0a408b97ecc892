"""The arena-words converter (csrc/mjx_selfplay.cuh) on the host build: on emulated self-play games and on hand-built games holding
every event type, its arrays equal dataset_codec.encode_events over the events mjai_log.decode_events reads from the words (with
start_game / end_game around them, augment_events when augmenting), plus their deltas and line numbers; corrupt words and
overflowed logs get their status and no entries, and no store passes a capacity."""
import numpy as np
import pytest

import emul_lib as E
import test_emul_mjai_write as MW
from mortal_b200 import _cdecl, dataset_codec, mjai_log
from mortal_b200.dataset_codec import HORA_WORDS, KYOKU_WORDS

_HEADER = open(_cdecl.HEADER.replace("mjx.h", "mjx_selfplay.h")).read()
OK, CORRUPT, CAPACITY = (_cdecl.enum(_HEADER, "mjx_aw_status")[k] for k in ("MJX_AW_OK", "MJX_AW_CORRUPT", "MJX_AW_CAPACITY"))
SENTINEL = 0xA5A5A5A5A5A5A5A5
GUARD = 64  # words (entries) past every capacity that must stay untouched


def convert(words, lens, augment=False, log_cap=None, short=0):
    """emulsp_convert count + fill -> (counts int32 [n, 4], per game None or dict(hdr, lines, kyoku [k, 19], hora [h, 2], deltas
    [n_ev, 4], has [n_ev])). `short` shrinks every capacity argument by that many entries below what the counts ask for; the
    arrays carry GUARD more entries, which must keep the sentinel."""
    L = E.lib()
    words = np.ascontiguousarray(words, dtype=np.uint64)
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    n, pitch = words.shape
    log_cap = pitch if log_cap is None else log_cap
    counts = np.full((n, 4), -7, dtype=np.int32)
    assert L.emulsp_convert(n, words.ctypes.data, lens.ctypes.data, pitch, log_cap, int(augment), counts.ctypes.data, None, None, None,
                            None, None, 0, None, 0, None, 0, None, None) == 0
    excl = lambda x: (np.cumsum(x) - x).astype(np.int32)
    ev_off, ky_off, ho_off = excl(counts[:, 1]), excl(counts[:, 2]), excl(counts[:, 3])
    n_ev, n_ky, n_ho = (int(counts[:, k].sum()) for k in (1, 2, 3))
    c_ev, c_ky, c_ho = max(n_ev - short, 0), max(n_ky - short, 0), max(n_ho - short, 0)
    hdr = np.full(n_ev + GUARD, SENTINEL, dtype=np.uint64)
    lines = np.full(n_ev + GUARD, -1, dtype=np.int32)
    kyoku = np.full((n_ky + GUARD) * KYOKU_WORDS, SENTINEL, dtype=np.uint64)
    hora = np.full((n_ho + GUARD) * HORA_WORDS, SENTINEL, dtype=np.uint64)
    deltas = np.full((n_ev + GUARD, 4), -7, dtype=np.int32)
    has = np.zeros(n_ev + GUARD, dtype=np.uint8)
    assert L.emulsp_convert(n, words.ctypes.data, lens.ctypes.data, pitch, log_cap, int(augment), counts.ctypes.data,
                            ev_off.ctypes.data, ky_off.ctypes.data, ho_off.ctypes.data, hdr.ctypes.data, lines.ctypes.data, c_ev,
                            kyoku.ctypes.data, c_ky * KYOKU_WORDS, hora.ctypes.data, c_ho * HORA_WORDS, deltas.ctypes.data,
                            has.ctypes.data) == 0
    assert (hdr[c_ev:] == SENTINEL).all() and (lines[c_ev:] == -1).all() and (deltas[c_ev:] == -7).all() and not has[c_ev:].any()
    assert (kyoku[c_ky * KYOKU_WORDS:] == SENTINEL).all() and (hora[c_ho * HORA_WORDS:] == SENTINEL).all()
    out = []
    for g in range(n):
        if counts[g, 0] != OK:
            assert tuple(counts[g, 1:]) == (0, 0, 0)
            out.append(None)
            continue
        e, k, h = slice(ev_off[g], ev_off[g] + counts[g, 1]), slice(ky_off[g], ky_off[g] + counts[g, 2]), slice(ho_off[g], ho_off[g] + counts[g, 3])
        out.append(dict(hdr=hdr[e], lines=lines[e], kyoku=kyoku.reshape(-1, KYOKU_WORDS)[k], hora=hora.reshape(-1, HORA_WORDS)[h],
                        deltas=deltas[e], has=has[e]))
    return counts, out


def reference(words, length, augment=False):
    """the arrays of the game's written file: decode_events + start_game / end_game, augment_events, encode_events with hora"""
    events = [{"type": "start_game", "names": ["a", "b", "c", "d"], "seed": [1, 2]}]
    events += mjai_log.decode_events(words[:length]) + [{"type": "end_game"}]
    if augment:
        events = dataset_codec.augment_events(events)
    hora = []
    hdr, pay = dataset_codec.encode_events(events, hora=hora)
    dl = [(ev["deltas"], True) if ev["type"] in ("hora", "ryukyoku") else None for ev in events]
    return dict(hdr=hdr, lines=np.arange(1, len(events) + 1, dtype=np.int32), kyoku=pay,
                hora=np.array(hora, dtype=np.uint64).reshape(-1, HORA_WORDS), deltas=dl)


def check_game(got, ref):
    assert got is not None
    np.testing.assert_array_equal(got["hdr"], ref["hdr"])
    np.testing.assert_array_equal(got["lines"], ref["lines"])
    np.testing.assert_array_equal(got["kyoku"], ref["kyoku"])
    np.testing.assert_array_equal(got["hora"], ref["hora"])
    for e, d in enumerate(ref["deltas"]):
        if d is None:
            assert got["has"][e] == 0  # the entries of other events are not written
        else:
            assert got["has"][e] == 1 and list(got["deltas"][e]) == list(d[0]), e


def emul_games(n, seed, policy_kind, cap=8192):
    nonces = np.arange(7000 + 37 * seed, 7000 + 37 * seed + n, dtype=np.uint64)
    env = E.EmulEnv(nonces, np.full(n, 11 + seed, dtype=np.uint64), enable_quick_eval=bool(seed % 2 == 0))
    env.enable_log(cap)
    acts = None
    while True:
        env.step(acts)
        if env.num_rows() == 0 and env.num_live() == 0:
            break
        acts = env.policy_test(policy_kind)
    words, lens = env.read_log()
    env.close()
    return words, lens


@pytest.mark.parametrize("seed,policy_kind", [(0, 1), (1, 0), (2, 2), (3, 1)])
@pytest.mark.parametrize("augment", [False, True])
def test_selfplay_games_equal_the_written_files(seed, policy_kind, augment):
    words, lens = emul_games(6, seed, policy_kind)
    counts, got = convert(words, lens, augment)
    assert (counts[:, 0] == OK).all()
    types = np.zeros(17, dtype=np.int64)
    for g in range(len(lens)):
        ref = reference(words[g], int(lens[g]), augment)
        check_game(got[g], ref)
        assert tuple(counts[g, 1:]) == (len(ref["hdr"]), len(ref["kyoku"]), len(ref["hora"]))
        types += np.bincount(ref["hdr"].astype(np.int64) & 0xFF, minlength=17)
    assert types[dataset_codec.START_KYOKU] >= 6 * 4
    assert types[dataset_codec.HORA] > 0 or policy_kind == 0  # the uniform random policy rarely wins a hand


@pytest.mark.parametrize("augment", [False, True])
def test_every_event_type(augment):
    """hand-built games: every event type, red fives, a round whose number differs from its dealer, 5-marker ura, double ron"""
    words, lens, _ = MW.synthetic_batch(4, 4, np.random.default_rng(17 + augment))
    counts, got = convert(words, lens, augment)
    assert (counts[:, 0] == OK).all()
    for g in range(4):
        ref = reference(words[g], int(lens[g]), augment)
        check_game(got[g], ref)
        assert set(int(x) & 0xFF for x in ref["hdr"]) == set(range(1, 17))


def test_pitch_wider_than_capacity():
    words, lens = emul_games(3, 5, 1)
    wide = np.full((3, words.shape[1] + 40), SENTINEL, dtype=np.uint64)
    wide[:, :words.shape[1]] = words
    counts, got = convert(wide, lens, log_cap=words.shape[1])
    for g in range(3):
        check_game(got[g], reference(words[g], int(lens[g])))


@pytest.mark.parametrize("cls,at,word,new_len", MW._corrupt_cases())
def test_corrupt_words_get_corrupt_and_no_entries(cls, at, word, new_len):
    words, lens, _ = MW.synthetic_batch(3, 4, np.random.default_rng(3))
    g = 1
    if cls == "ura_38":
        at = int(np.nonzero((words[g] & 0xFF) == mjai_log.HORA)[0][0])
    if cls == "truncated_hora":
        lens[g] = int(np.nonzero((words[g] & 0xFF) == mjai_log.HORA)[0][0]) + 2
    elif new_len is not None:
        lens[g] = new_len
    if at is not None:
        words[g, at] = word
    with pytest.raises((ValueError, IndexError)):
        mjai_log.decode_events(words[g, :int(lens[g])])
    counts, got = convert(words, lens)
    assert list(counts[:, 0]) == [OK, CORRUPT, OK] and got[1] is None
    for k in (0, 2):  # the games around it are placed as if the corrupt one were absent
        check_game(got[k], reference(words[k], int(lens[k])))


def test_overflowed_log_gets_capacity_and_reads_stay_inside():
    words, lens, _ = MW.synthetic_batch(3, 4, np.random.default_rng(5))
    lens[0] = words.shape[1] + 100
    lens[2] = -3
    counts, got = convert(words, lens)
    assert list(counts[:, 0]) == [CAPACITY, OK, CAPACITY]
    check_game(got[1], reference(words[1], int(lens[1])))
    counts, _ = convert(words[:, :40], np.full(3, 41, dtype=np.int32), log_cap=40)  # the arena log overflowed by one word
    assert (counts[:, 0] == CAPACITY).all()


@pytest.mark.parametrize("short", [1, 3])
def test_short_capacities_write_nothing_past_them(short):
    words, lens = emul_games(4, 7, 1)
    convert(words, lens, short=short)  # convert() checks the guard regions
