"""Replays the reference's only seeded full-game log through the oracle, end to end.

Fixture: tests/golden/golden_game.jsonl, extracted by tools/extract_ref_fixtures.py from
Mortal's log-viewer/index.example.html:10-264 (seed [10637, 12210010324280706444]).
Pins: SHA3/ChaCha12/rand-0.8 shuffle + wall slicing (every haipai, tsumo, dora, ura marker),
PlayerState legal-action masks (`meta.mask_bits` of every logged decision), riichi sticks,
honba/kyotaku payout, hora deltas, scores at each start_kyoku and the tobi ending.
"""
import ctypes as C
import json
import os

import numpy as np

import oracle_lib as O

HERE = os.path.dirname(os.path.abspath(__file__))
AGENT_EVENTS = {"dahai", "chi", "pon", "daiminkan", "kakan", "ankan", "reach"}


def load_golden():
    with open(os.path.join(HERE, "golden", "golden_game.jsonl")) as f:
        return [json.loads(ln) for ln in f if ln.strip()]


def strip_meta(ev):
    return {k: v for k, v in ev.items() if k != "meta"}


def oracle_log(L, g):
    buf = (O.OrcEvent * 4096)()
    n = L.orc_game_log(g, buf, 4096)
    assert n <= 4096
    return [O.event_to_dict(buf[i]) for i in range(n)]


def test_golden_game_replay():
    L = O.lib()
    golden = load_golden()
    assert golden[0]["type"] == "start_game" and golden[0]["seed"] == [10637, 12210010324280706444]
    events = [e for e in golden[1:] if e["type"] != "end_game"]
    nonce, key = golden[0]["seed"]
    g = L.orc_game_new(nonce, key, 1, 0)  # shuffle_kind 1 = rand 0.8
    try:
        checked_masks = 0
        for _ in range(10000):
            ended = L.orc_game_poll(g)
            assert ended >= 0, O.err()
            log = oracle_log(L, g)
            # everything the oracle emitted so far must equal the golden prefix
            assert len(log) <= len(events)
            for i, (a, b) in enumerate(zip(log, events)):
                assert a == strip_meta(b), (i, a, strip_meta(b))
            if ended:
                break
            nxt = events[len(log)]
            acting = []
            for seat in range(4):
                ps = O.PlayerState(0, _ptr=L.orc_game_state(g, seat), _own=False)
                if O.unpack_cans(ps.view().cans) and any(
                    O.unpack_cans(ps.view().cans)[k] for k in O.CAN_BITS
                ):
                    acting.append((seat, ps))
            assert acting, "poll returned in-game with nobody able to act"
            if nxt["type"] in AGENT_EVENTS:
                actor = nxt["actor"]
                assert actor in [s for s, _ in acting]
                ps = dict(acting)[actor]
                meta = nxt.get("meta")
                if meta and "mask_bits" in meta:
                    mask = ps.legal_mask(False)
                    bits = sum(1 << i for i in range(46) if mask[i])
                    assert bits == meta["mask_bits"], (len(log), nxt, bin(bits), bin(meta["mask_bits"]))
                    checked_masks += 1
                    if "kan_select" in meta:
                        kmask = ps.legal_mask(True)
                        kbits = sum(1 << i for i in range(46) if kmask[i])
                        assert kbits == meta["kan_select"]["mask_bits"]
                e = O.event_from_json(strip_meta(nxt))
                L.orc_game_set_reaction(g, actor, C.byref(e))
            elif nxt["type"] == "hora":
                j = len(log)
                while events[j]["type"] == "hora":
                    h = events[j]
                    assert h["actor"] in [s for s, _ in acting]
                    e = O.event_from_json({"type": "hora", "actor": h["actor"], "target": h["target"]})
                    L.orc_game_set_reaction(g, h["actor"], C.byref(e))
                    j += 1
            elif nxt["type"] == "ryukyoku":
                seat = [s for s, ps in acting if O.unpack_cans(ps.view().cans)["can_ryukyoku"]]
                assert seat, "ryukyoku in golden log but nobody can declare it"
                e = O.event_from_json({"type": "ryukyoku"})
                L.orc_game_set_reaction(g, seat[0], C.byref(e))
            else:
                # everybody passed: next golden event is board-generated (tsumo / reach_accepted / dora)
                assert nxt["type"] in ("tsumo", "reach_accepted", "dora"), nxt
            L.orc_game_advance_step(g)
        else:
            raise AssertionError("game did not end")
        log = oracle_log(L, g)
        assert len(log) == len(events)
        assert checked_masks >= 100
        scores = np.zeros(4, dtype=np.int32)
        assert L.orc_game_finish(g, scores.ctypes.data) == 0, O.err()
        # last kyoku: scores at start [32700,30200,13100,24000] + deltas [0,20000,-18000,0] -> tobi
        assert list(scores) == [32700, 49200, -5900, 24000]  # seats 1 and 2 each paid a riichi stick; sum 100000
        info = np.zeros(9, dtype=np.int32)
        L.orc_game_info(g, info.ctypes.data)
        assert info[7] == 1 and info[8] == 3
    finally:
        L.orc_game_free(g)


def test_wall_layout_matches_golden_haipai():
    """board.rs:109-122 slicing + UNSHUFFLED aka placement, against the three golden start_kyoku events."""
    L = O.lib()
    golden = load_golden()
    nonce, key = golden[0]["seed"]
    starts = [e for e in golden if e["type"] == "start_kyoku"]
    for sk, (kyoku, honba) in zip(starts, [(0, 0), (0, 1), (1, 0)]):
        seq = np.zeros(136, dtype=np.uint8)
        L.orc_make_wall(nonce, key, kyoku, honba, 1, seq.ctypes.data)
        assert sorted(seq.tolist()) == sorted([t for t in range(34) for _ in range(4) if t not in (4, 13, 22)]
                                              + [4] * 3 + [13] * 3 + [22] * 3 + [34, 35, 36])
        for seat in range(4):
            assert [O.TILE_NAMES[t] for t in seq[13 * seat: 13 * seat + 13]] == sk["tehais"][seat]
        assert O.TILE_NAMES[seq[60]] == sk["dora_marker"]


def test_sha3_and_chacha_known_answers():
    """FIPS 202 SHA3-256("") and RFC 7539-style ChaCha block structure (12 rounds, zero key)."""
    L = O.lib()
    out = np.zeros(32, dtype=np.uint8)
    L.orc_sha3_256(None, 0, out.ctypes.data)
    assert out.tobytes().hex() == "a7ffc6f8bf1ed76651c14756a061d662f580ff4de43b49fa82d80a4b80f8434a"
    import hashlib
    msg = bytes(range(200))
    m = np.frombuffer(msg, dtype=np.uint8).copy()
    L.orc_sha3_256(m.ctypes.data, len(msg), out.ctypes.data)
    assert out.tobytes() == hashlib.sha3_256(msg).digest()
    # rand_chacha ChaCha12Rng::from_seed([0;32]) first word (published test vector of chacha12, zero key/nonce)
    seed = np.zeros(32, dtype=np.uint8)
    w = np.zeros(32, dtype=np.uint32)
    L.orc_chacha12(seed.ctypes.data, w.ctypes.data, 32)
    # ChaCha12 zero key, zero counter keystream begins 9b f4 9a 6a 07 55 f9 53 ...
    assert w[:2].tobytes().hex() == "9bf49a6a0755f953"
    assert len(set(w.tolist())) == 32


def test_rand09_shuffle_is_a_permutation_and_differs():
    L = O.lib()
    a = np.zeros(136, dtype=np.uint8)
    b = np.zeros(136, dtype=np.uint8)
    L.orc_make_wall(10000, 0x2000, 0, 0, 0, a.ctypes.data)
    L.orc_make_wall(10000, 0x2000, 0, 0, 1, b.ctypes.data)
    assert sorted(a.tolist()) == sorted(b.tolist())
    assert a.tolist() != b.tolist()


def test_gameplay_loader_restatement_on_golden_log():
    """The oracle's restatement of dataset/gameplay.rs is pinned to the reference's own data: on the seeded example log
    every non-pass move it extracts is, in order, exactly the agent event the log holds for that player (dahai / reach /
    chi / pon), and where the log carries the agent's `meta.mask_bits` (written by the reference itself) the extracted
    legal mask equals it."""
    golden = load_golden()
    events = [strip_meta(e) for e in golden]
    tile_id = {name: i for i, name in enumerate(O.TILE_NAMES)}
    checked_masks = 0
    for p in range(4):
        got = O.gameplay_load(events, p, with_obs=False, sp_mode=0)
        # pass (45) has no event at all; agari (43) shows up as the board's `hora`, not as an agent event
        moves = [(int(a), got["masks"][i]) for i, a in enumerate(got["actions"]) if a not in (43, 45)]
        n_hora = sum(e["type"] == "hora" and e["actor"] == p for e in golden)
        assert int((got["actions"] == 43).sum()) == n_hora, (p, n_hora)
        logged = [e for e in golden if e.get("actor") == p and e["type"] in AGENT_EVENTS]
        assert len(moves) == len(logged) and len(moves) > 20, (p, len(moves), len(logged))
        for (label, mask), e in zip(moves, logged):
            if e["type"] == "dahai":
                assert label == tile_id[e["pai"]], (p, e, label)
            elif e["type"] == "reach":
                assert label == 37
            elif e["type"] == "pon":
                assert label == 41
            elif e["type"] == "chi":
                assert label in (38, 39, 40)
            if "meta" in e and "mask_bits" in e["meta"]:
                assert sum(1 << i for i in range(46) if mask[i]) == e["meta"]["mask_bits"], (p, e)
                checked_masks += 1
        # bookkeeping columns: kyoku index non-decreasing from 0 to 2, apply_gamma exactly on discards / riichi / kans
        assert got["at_kyoku"][0] == 0 and got["at_kyoku"][-1] == 2 and (np.diff(got["at_kyoku"].astype(int)) >= 0).all()
        assert (got["apply_gamma"] == (got["actions"] <= 37)).all()
    assert checked_masks >= 100
