"""The review on the host-emulated build (tests/host_emul/emul_review.cc: review mode of the replay, k_review_react's and
k_review_render's code on one host lane) against libriichi.mjai.Bot on the emulated PlayerState (emul_state.EmulStateBackend),
driven line by line as mortal.py's review mode drives it: byte for byte with meta.eval_time_ns masked (CPU only)."""
import json
import os

import numpy as np
import pytest

import review_lib
import validate_lib
import viewpoint_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_game.jsonl")


def _text(events):
    return "".join(json.dumps(e, separators=(",", ":")) + "\n" for e in events)


@pytest.fixture(scope="module")
def emul_bot():
    from emul_state import EmulStateBackend
    from mortal_b200.libriichi import state

    prev = state._backend
    state.set_backend(EmulStateBackend())
    yield
    state.set_backend(prev)


@pytest.fixture(scope="module")
def logs():
    """(events, seats): the golden game, emulated self-play games of both test-policy kinds, and their single-viewpoint versions
    for every seat"""
    out = [([json.loads(ln) for ln in open(GOLDEN) if ln.strip()], [0, 1, 2, 3])]
    for policy in (0, 1):
        games = validate_lib.emul_games(2, policy, seed0=771000 + 100 * policy)
        out += [(g, [0, 1, 2, 3]) for g in games]
        out += [(viewpoint_lib.viewpoint(games[0], p), [p]) for p in range(4)]
        out += review_lib.guard_logs(validate_lib.emul_games(4, policy, seed0=772000 + 100 * policy))
    return out


@pytest.mark.parametrize("guard", [True, False])
def test_emul_review_equals_the_bot(emul_bot, logs, guard):
    engine = review_lib.StubEngine(guard)
    got = review_lib.emul_review(engine, [ev for ev, _ in logs], [s for _, s in logs])
    jobs = [(ev, p) for ev, ps in logs for p in ps]
    texts = []
    for (ev, p), (text, rec, err, stop) in zip(jobs, got):
        assert err == 0 and stop == len(ev)
        want = review_lib.bot_review(engine, _text(ev), p)
        assert review_lib.mask_eval(text) == review_lib.mask_eval(want)
        assert text.count("\n") == len(ev)
        texts.append(text)
    text = "".join(texts)
    for kind in ("dahai", "chi", "pon", "reach", "hora", "ankan", "kakan"):
        assert f'{{"type":"{kind}"' in text, kind
    assert '{"type":"none","meta":{"q_values"' in text  # a pass
    assert review_lib.NONE_LINE in text
    lines = text.splitlines()
    assert any(ln.startswith('{"type":"ankan"') and '"kan_select":{' in ln for ln in lines)
    assert any(ln.startswith('{"type":"kakan"') and '"kan_select":{' in ln for ln in lines)
    main = [r for _, r, _, _ in got]
    labels = np.concatenate([r["info"][r["kan"] == 0, 3] for r in main])
    assert (labels >= 0).any() and (labels < 0).any()
    over = sum(int(((r["engine_action"] == 43) & (r["info"][:, 0] != 43) & (r["kan"] == 0)).sum()) for r in main)
    assert (over > 0) == guard


def test_emul_review_errors(emul_bot, logs):
    """a reaction that cannot be decoded fails that job alone, at the event where the Bot raises; a log hiding the seat's own tiles
    fails with 13 before its first event is applied"""
    engine = review_lib.IllegalStubEngine(True)
    full, vp = logs[1][0], logs[3][0]  # a full-information log; seat 0's viewpoint
    got = review_lib.emul_review(engine, [full, vp, vp], [[0, 1, 2, 3], [1], [0]])
    failed = 0
    for p in range(4):
        text, _, err, stop = got[p]
        at = review_lib.bot_fail_index(engine, _text(full), p)
        if at is None:
            assert err == 0 and review_lib.mask_eval(text) == review_lib.mask_eval(review_lib.bot_review(engine, _text(full), p))
        else:
            assert text is None and err == 1 and stop == at  # ERR_ILLEGAL_ACTION, at the Bot's event
            failed += 1
    assert failed > 0
    assert got[4][0] is None and got[4][2] == 13 and got[4][3] == 0
    assert got[5][2] == 0 or got[5][3] == review_lib.bot_fail_index(engine, _text(vp), 0)
