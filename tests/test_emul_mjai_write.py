"""The mjai log renderer (csrc/mjx_mjai_write.cuh) on the host build: its Q-value formatter against CPython's float repr, and the
rendered text against the host writer (mortal_b200/mjai_log.py decode_events + attach_meta + dump_json_log) on emulated self-play
games and on hand-built games that hold every event type, every meta variant and every corrupt-word class."""
import struct

import numpy as np
import pytest
import torch

import emul_lib as E
import mjai_write_lib as W
from mortal_b200 import mjai_log, mjai_write
from mortal_b200.libriichi.arena import _MetaRecorder

NAMES = ["Ｍortal", "café", "名前", 'a"b\\c']


# ---- formatter ------------------------------------------------------------------------------------------------------------------
def _repr_json(bits):
    f = np.asarray(bits, dtype=np.uint32).view(np.float32).astype(np.float64).tolist()
    return ["NaN" if x != x else "Infinity" if x == float("inf") else "-Infinity" if x == -float("inf") else repr(x) for x in f]


def test_formatter_examples():
    vals = np.array([0.1, -1.7, 1.0, 123456792.0, 9.999999747378752e-06, 1.0000000272564224e+16, 1.401298464324817e-45, -0.0, 0.0,
                     float("nan"), float("inf"), -float("inf"), np.finfo(np.float32).max, -np.finfo(np.float32).tiny], dtype=np.float32)
    assert W.format_f32(vals) == ["0.10000000149011612", "-1.7000000476837158", "1.0", "123456792.0", "9.999999747378752e-06",
                                  "1.0000000272564224e+16", "1.401298464324817e-45", "-0.0", "0.0", "NaN", "Infinity", "-Infinity",
                                  "3.4028234663852886e+38", "-1.1754943508222875e-38"]


def test_formatter_every_exponent_edges_against_cpython():
    """every f32 exponent (both signs) with its first and last 4,096 mantissas, through PyOS_double_to_string"""
    for sign in (0, 1):
        for ex in range(256):
            base = (sign << 31) | (ex << 23)
            for lo in (base, base + (1 << 23) - 4096):
                bad, first = W.sweep(lo, lo + 4096)
                assert bad == 0, f"{bad} mismatches, first {first:#010x}"


def test_formatter_random_patterns_and_specials_against_cpython():
    """2^24 random bit patterns through PyOS_double_to_string, and ±0, subnormals, FLT_MAX, NaN and ±inf against json's text"""
    special = np.array([0, 1 << 31, 1, 0x807FFFFF, 0x007FFFFF, 0x00800000, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F800000, 0xFF800000, 0x7FC00000,
                        0xFFC00001, 0x7F800001], dtype=np.uint32)
    assert W.format_f32(special) == _repr_json(special)
    bits = np.random.default_rng(7).integers(0, 1 << 32, size=1 << 24, dtype=np.uint64).astype(np.uint32)
    assert W.format_f32(bits[:100000]) == _repr_json(bits[:100000])
    bad, first = W.check(bits)
    assert bad == 0, f"{bad} mismatches, first {first:#010x}"


# ---- rendering ------------------------------------------------------------------------------------------------------------------
def host_text(words, lens, g, bounds, decisions, names, seed):
    events, offs = mjai_log.decode_events(words[g, :int(lens[g])], with_offsets=True)
    if bounds is not None and decisions is not None:
        mjai_log.attach_meta(events, offs, [int(b) for b in bounds[:, g]], decisions[g])
    return mjai_log.dump_json_log(events, names, seed).encode("utf-8")


def device_texts(words, lens, rec, names, seeds):
    bounds = recs = None
    if rec is not None:
        bounds, recs = mjai_write.recorder_records(rec)
    status, texts = W.render(words, lens, bounds, recs)
    heads = mjai_write._heads([names] * len(seeds), seeds)
    return status, [None if t is None else h + t + e for t, (h, e) in zip(texts, heads)]


def compare(words, lens, rec, n):
    seeds = [(1000 + g, 7) for g in range(n)]
    status, got = device_texts(words, lens, rec, NAMES, seeds)
    assert (status == 0).all(), status
    bounds = decisions = None
    if rec is not None:
        bounds, decisions = rec.finish()
    n_meta = n_kan = 0
    for g in range(n):
        ref = host_text(words, lens, g, bounds, decisions, NAMES, seeds[g])
        assert got[g] == ref, _first_diff(got[g], ref)
        n_meta += ref.count(b'"meta"')
        n_kan += ref.count(b'"kan_select"')
    return n_meta, n_kan


def _first_diff(a, b):
    la, lb = a.split(b"\n"), b.split(b"\n")
    for i, (x, y) in enumerate(zip(la, lb)):
        if x != y:
            return f"line {i}:\n  device {x[:400]!r}\n  host   {y[:400]!r}"
    return f"line counts {len(la)} != {len(lb)}"


def selfplay(n, version, greedy_mode, q_kind, seed, dev_rec=None):
    """emulated self-play with a recorder fed exactly as _Part.decide feeds it; dev_rec (mjai_write_lib.EmulRecords) also gets
    every agent call as DeviceMetaRecorder.record hands it to k_meta_record"""
    rng = np.random.default_rng(seed)
    nonces = np.arange(5100 + 10 * seed, 5100 + 10 * seed + n, dtype=np.uint64)
    env = E.EmulEnv(nonces, np.full(n, 3, dtype=np.uint64), enable_quick_eval=True)
    env.enable_log()
    rec = _MetaRecorder(n, version)
    acts, cycles = None, 0
    while True:
        env.step(acts)
        rec.add_bounds(torch.from_numpy(env.log_lens()))
        rt, rs, masks = env.rows()
        nr = len(rt)
        if nr == 0 and env.num_live() == 0:
            break
        acts = env.policy_test(1)
        if nr:
            obs = torch.from_numpy(env.encode_obs(sp=False, version=4))
            q = torch.from_numpy(rng.standard_normal((nr, 46)).astype(np.float32))
            if q_kind == "special":
                q[torch.from_numpy(rng.random((nr, 46)) < 0.05)] = float("nan")
                q[torch.from_numpy(rng.random((nr, 46)) < 0.05)] = -float("inf")
                q[torch.from_numpy(rng.random((nr, 46)) < 0.05)] = 0.1
            half = nr // 2
            for idx in (torch.arange(half), torch.arange(half, nr)):  # two agent calls, as with a challenger and a champion
                if idx.numel():
                    g = None if greedy_mode is None else torch.from_numpy(rng.random(idx.numel()) < 0.7)
                    ns = int(rng.integers(1, 10 ** 9))
                    rec.add_agent(cycles, idx, q[idx], ns, g)
                    if dev_rec is not None:  # the device recorder's kernel on the same call
                        dev_rec.calls.append((idx.numel(), ns))
                        dev_rec.record(cycles, q[idx].numpy(), rt, rs, acts, masks, idx=idx.numpy(), greedy=None if g is None else g.numpy(),
                                       call=len(dev_rec.calls) - 1, obs=obs.numpy() if version == 4 else None)
            rec.add_rows(cycles, torch.from_numpy(rt).long(), torch.from_numpy(rs), torch.from_numpy(acts[:nr]), torch.from_numpy(masks),
                         obs)
        cycles += 1
    words, lens = env.read_log()
    env.close()
    return words, lens, rec


@pytest.mark.parametrize("version,greedy,q_kind", [(4, None, "normal"), (4, "flags", "special"), (0, "flags", "normal")])
def test_selfplay_logs_equal_the_host_writer(version, greedy, q_kind):
    n = 8
    words, lens, rec = selfplay(n, version, greedy, q_kind, seed=version + (greedy is not None))
    n_meta, _ = compare(words, lens, rec, n)
    assert n_meta > 8 * 150
    compare(words, lens, None, n)  # log_meta=False


@pytest.mark.parametrize("version,greedy", [(4, "flags"), (0, None)])
def test_device_recorder_records_render_as_the_host_recorder(version, greedy):
    """k_meta_record (host build) fed every agent call: its records render exactly as _MetaRecorder's through the host writer"""
    n = 8
    dev = W.EmulRecords(1 << 17)
    words, lens, rec = selfplay(n, version, greedy, "special", seed=20 + version, dev_rec=dev)
    assert dev.count < dev.cap
    bounds = np.array(rec.bounds, dtype=np.int32)
    status, texts = W.render(words, lens, bounds, dev.render_recs())
    assert (status == 0).all()
    hb, decisions = rec.finish()
    heads = mjai_write._heads([NAMES] * n, [(1000 + g, 7) for g in range(n)])
    n_meta = 0
    for g in range(n):
        ref = host_text(words, lens, g, hb, decisions, NAMES, (1000 + g, 7))
        got = heads[g][0] + texts[g] + heads[g][1]
        assert got == ref, _first_diff(got, ref)
        n_meta += ref.count(b'"meta"')
    assert n_meta > 8 * 150


# ---- hand-built games -----------------------------------------------------------------------------------------------------------
M32 = 0xFFFFFFFF


def wd(ty, actor=0, target=0, pai=37, tg=0, aux=0, c=(0, 0, 0, 0), extra=0):
    return (ty | actor << 8 | target << 10 | pai << 12 | tg << 20 | aux << 21 | c[0] << 24 | c[1] << 32 | c[2] << 40 | c[3] << 48
            | extra << 56)


def i4(v):
    return [(v[0] & M32) | (v[1] & M32) << 32, (v[2] & M32) | (v[3] & M32) << 32]


def haipai(rng):
    raw = bytes(int(x) for x in rng.integers(0, 38, size=52)) + b"\0" * 4
    return list(struct.unpack("<7Q", raw))


def synthetic_game(rng):
    """[(words, actor, [(seat, kan, action)] rows decided one step before the event)] covering every event type"""
    T = mjai_log
    ev = []
    ev.append(([wd(T.START_KYOKU, pai=int(rng.integers(38)), c=(5, 2, 3, 1))] + i4([-1200, 35000, 25000, 41200]) + haipai(rng), 0, []))
    ev.append(([wd(T.TSUMO, 1, pai=5)], 1, [(1, 0, 45)]))
    ev.append(([wd(T.DAHAI, 1, pai=36, tg=1)], 1, [(1, 0, 36), (2, 0, 45)]))
    ev.append(([wd(T.CHI, 2, 1, pai=36, c=(3, 5, 0, 0))], 2, [(2, 0, 39), (3, 0, 45)]))
    ev.append(([wd(T.DAHAI, 2, pai=0)], 2, [(2, 0, 0)]))
    ev.append(([wd(T.PON, 0, 2, pai=0, c=(0, 0, 0, 0))], 0, [(0, 0, 41)]))
    ev.append(([wd(T.DAHAI, 0, pai=9)], 0, [(0, 0, 7)]))  # action does not produce this dahai: no meta
    ev.append(([wd(T.DAIMINKAN, 3, 0, pai=9, c=(9, 9, 9, 0))], 3, [(3, 0, 42)]))
    ev.append(([wd(T.DORA, pai=33)], 0, []))
    ev.append(([wd(T.KAKAN, 3, pai=27, c=(27, 27, 27, 0))], 3, [(3, 0, 42), (3, 1, 27)]))  # kan_select nested
    ev.append(([wd(T.ANKAN, 1, c=(31, 31, 31, 31))], 1, [(1, 1, 31), (1, 0, 42)]))
    ev.append(([wd(T.ANKAN, 2, c=(30, 30, 30, 30))], 2, [(2, 1, 30)]))  # a kan-select row without its main row: no meta
    ev.append(([wd(T.REACH, 0)], 0, [(0, 0, 37), (0, 0, 37)]))  # two rows with one key: the last one counts
    ev.append(([wd(T.DAHAI, 0, pai=12)], 0, [(0, 0, 12)]))
    ev.append(([wd(T.REACH_ACCEPTED, 0)], 0, []))
    ev.append(([wd(T.HORA, 1, 0, aux=5, c=(1, 2, 3, 4), extra=37)] + i4([-8000, 8000, 0, 0]), 1, [(1, 0, 43), (2, 0, 43)]))
    ev.append(([wd(T.HORA, 2, 0, aux=0)] + i4([-3900, 0, 3900, 0]), 2, "same"))  # double ron: both written by one step
    ev.append(([wd(T.END_KYOKU)], 0, []))
    ev.append(([wd(T.START_KYOKU, pai=4, c=(12, 0, 0, 0))] + i4([0, 0, -100, 100]) + haipai(rng), 0, []))
    ev.append(([wd(T.TSUMO, 0, pai=27)], 0, []))
    ev.append(([wd(T.RYUKYOKU)] + i4([0, 0, 0, 0]), 0, [(1, 0, 45), (0, 0, 44)]))  # kyushu: the seat whose action is 44
    ev.append(([wd(T.END_KYOKU)], 0, []))
    ev.append(([wd(T.START_KYOKU, pai=4, c=(1, 1, 0, 0))] + i4([0, 0, 0, 0]) + haipai(rng), 0, []))
    ev.append(([wd(T.RYUKYOKU)] + i4([3000, -1000, -1000, -1000]), 0, [(0, 0, 45)]))  # exhaustive: nobody declared it
    ev.append(([wd(T.END_KYOKU)], 0, []))
    return ev


def synthetic_batch(n, version, rng, corrupt=None):
    games = [synthetic_game(rng) for _ in range(n)]
    cap = max(sum(len(w) for w, _, _ in g) for g in games) + 4
    words = np.zeros((n, cap), dtype=np.uint64)
    lens = np.zeros(n, dtype=np.int32)
    n_steps = max(len(g) for g in games)
    bounds = np.zeros((n_steps, n), dtype=np.int32)
    rows = [[] for _ in range(n_steps)]  # per cycle: (table, seat, kan, action)
    for t, g in enumerate(games):
        at, k = 0, -1
        for w, actor, decided in g:
            if decided != "same":  # every event is written by a step of its own, except "same": by the step before's
                k += 1
            words[t, at:at + len(w)] = w
            at += len(w)
            bounds[k:, t] = at
            for seat, kan, action in ([] if decided == "same" else decided):
                if k >= 1:
                    rows[k - 1].append((t, seat, kan, action))
        lens[t] = at
    rec = _MetaRecorder(n, version)
    for c in range(n_steps):
        rec.add_bounds(torch.from_numpy(bounds[c].copy()))
        if not rows[c]:
            continue
        perm = rng.permutation(len(rows[c]))  # rows of a cycle come in any table order
        rr = [rows[c][i] for i in perm]
        nr = len(rr)
        tbl = torch.tensor([r[0] for r in rr], dtype=torch.long)
        rs = torch.tensor([r[1] | (r[2] << 2) for r in rr], dtype=torch.uint8)
        act = torch.tensor([r[3] for r in rr], dtype=torch.int64)
        masks = torch.from_numpy(rng.random((nr, 46)) < 0.3)
        masks[torch.arange(nr), act] = True
        q = torch.from_numpy((rng.standard_normal((nr, 46)) * 10.0 ** rng.integers(-6, 18, size=(nr, 1))).astype(np.float32))
        q[torch.from_numpy(rng.random((nr, 46)) < 0.05)] = float("nan")
        q[torch.from_numpy(rng.random((nr, 46)) < 0.05)] = -float("inf")
        obs = torch.from_numpy(rng.integers(0, 2, size=(nr, 869, 1)).astype(np.float32))
        rec.add_agent(c, torch.arange(nr), q, int(rng.integers(1, 1 << 40)), torch.from_numpy(rng.random(nr) < 0.5))
        rec.add_rows(c, tbl, rs, act, masks, obs)
    return words, lens, rec


@pytest.mark.parametrize("version", [4, 0])
def test_every_event_type_and_meta_variant(version):
    rng = np.random.default_rng(11 + version)
    words, lens, rec = synthetic_batch(5, version, rng)
    n_meta, n_kan = compare(words, lens, rec, 5)
    assert n_kan == 5 * 2 and n_meta == 5 * 13
    compare(words, lens, None, 5)


def _corrupt_cases():
    """(class, word index to overwrite or None, new word, new length) for one hand-built game"""
    T = mjai_log
    return [
        ("type_zero", 10, 0, None), ("type_15", 10, 15, None), ("type_255", 10, 255, None),
        ("pai_38", 10, wd(T.TSUMO, 1, pai=38), None), ("dahai_pai_255", 11, wd(T.DAHAI, 1, pai=255), None),
        ("consumed_38", 12, wd(T.CHI, 2, 1, pai=36, c=(3, 38, 0, 0)), None),
        ("ura_38", None, wd(T.HORA, 1, 0, aux=5, c=(1, 2, 3, 4), extra=38), None),
        ("bakaze_past_north", 0, wd(T.START_KYOKU, pai=1, c=(44, 0, 0, 0)), None),
        ("haipai_38", 5, 38, None),
        ("truncated_start_kyoku", None, None, 6), ("truncated_hora", None, None, -1),
    ]


@pytest.mark.parametrize("cls,at,word,new_len", _corrupt_cases())
def test_corrupt_words_get_a_status_and_the_host_raises(cls, at, word, new_len):
    rng = np.random.default_rng(3)
    words, lens, rec = synthetic_batch(2, 4, rng)
    g = 1
    if cls == "ura_38":
        at = int(np.nonzero((words[g] & 0xFF) == mjai_log.HORA)[0][0])
    if cls == "truncated_hora":
        hora = int(np.nonzero((words[g] & 0xFF) == mjai_log.HORA)[0][0])
        lens[g] = hora + 2
    elif new_len is not None:
        lens[g] = new_len
    if at is not None:
        words[g, at] = word
    status, _ = device_texts(words, lens, rec, NAMES, [(1, 2), (3, 4)])
    assert status[0] == 0 and status[1] != 0
    with pytest.raises((ValueError, IndexError)):
        mjai_log.decode_events(words[g, :int(lens[g])])


def test_log_longer_than_capacity_is_declined_and_reads_stay_inside():
    rng = np.random.default_rng(5)
    words, lens, rec = synthetic_batch(2, 4, rng)
    lens[0] = words.shape[1] + 100
    lens[1] = -3
    status, _ = device_texts(words, lens, rec, NAMES, [(1, 2), (3, 4)])
    assert list(status) == [3, 3]
