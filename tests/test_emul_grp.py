"""k_grp_logs's logic (csrc/mjx_grp.cuh, host build) against Grp.load_events: per log the feature rows, the ranking and the final
scores are equal, built as mortal_b200.dataset builds them from the kernel's outputs; the status is non-zero exactly where the host
raises. Also the shared read helpers of the device log readers."""
import json
import os

import numpy as np
import pytest

import grp_lib as G
import log_mutations as LM
from mortal_b200 import _logio, dataset_codec
from test_emul_stat import END, _dahai, _game, _hora, _reach, _ryu, _sk
from test_emul_vs_oracle import _selfplay_logs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _check(games):
    """every log: the Grp equals Grp.load_events, or the host raises and the status is non-zero with zeroed outputs"""
    a = G.encode(games)
    out = G.run_emul(a)
    _, rank, final, status = out
    for i, ev in enumerate(games):
        want = G.host_grp(ev)
        if isinstance(want, type):
            assert status[i] != 0, (i, want)
            assert not rank[i].any() and not final[i].any()
        else:
            assert status[i] == 0, (i, G.STATUS[int(status[i])])
            assert G.same(G.grp_of(a, out, i), want), i
    return status


def test_status_names():
    assert G.STATUS == {0: "OK", 1: "NO_DELTAS", 2: "NO_KYOKU", 3: "CAPACITY"}


def test_golden_game():
    with open(os.path.join(ROOT, "tests", "golden", "golden_game.jsonl")) as f:
        events = [json.loads(ln) for ln in f if ln.strip()]
    assert not _check([events]).any()


@pytest.fixture(scope="module")
def games():
    return _selfplay_logs(48, 1, 741000) + _selfplay_logs(24, 0, 742000)


def test_selfplay_logs(games):
    assert len(games) >= 64
    assert not _check(games).any()


def test_augmented_logs(games):
    aug = [dataset_codec.augment_events(ev) for ev in games[:24]]
    assert not _check(aug).any()


def test_mutation_corpus(games):
    corpus = LM.mutated_corpus(games, 6, np.random.default_rng(23))
    parsed = []
    for _, text in corpus:
        try:
            parsed.append([json.loads(ln) for ln in text.splitlines() if ln.strip()])
        except ValueError:  # `unparsable`: the host raises, the decoder declines; nothing reaches the kernel
            continue
    assert len(parsed) >= 6 * (len(LM.CLASSES) - 1)
    _check(parsed)


# ---- hand-built logs --------------------------------------------------------------------------------------------------------
def _round(bakaze, kyoku, honba=0, kyotaku=0, scores=(25000, 25000, 25000, 25000)):
    return dict(_sk(kyoku - 1, scores), bakaze=bakaze, kyoku=kyoku, honba=honba, kyotaku=kyotaku)


EDGE = {
    "east, south, west and north rounds": _game(*[[_round(w, k, honba=k - 1, kyotaku=k % 3), _dahai(0), _ryu([0, 0, 0, 0]), END]
                                                  for w in "ESWN" for k in (1, 4)]),
    "a tie stays in seat order": _game([_sk(2, (30000, 20000, 30000, 20000)), _dahai(2), _ryu([0, 0, 0, 0]), END]),
    "four equal final scores": _game([_sk(), _dahai(0), _ryu([0, 0, 0, 0]), END]),
    "a total under 100000 tops up the leader": _game([_sk(1, (30000, 30000, 20000, 19000)), _dahai(1), _ryu([0, 0, 0, 0]), END]),
    "sticks left on the table": _game([_sk(), *_reach(0), *_reach(3), _ryu([1500, -1500, -1500, 1500]), END]),
    "scores near the int32 limits": _game([_sk(0, (2147483647, 2147483647, -2147483648, -2147483648)), _dahai(0),
                                           _ryu([2147483647, 2147483647, -2147483648, -2147483648]), END]),
    "missing deltas in an earlier kyoku": _game([_sk(), _dahai(0), {"type": "hora", "actor": 1, "target": 0}, END],
                                                [_sk(1), _dahai(1), _hora(2, 1, [0, -3900, 3900, 0]), END]),
    "null deltas in an earlier kyoku": _game([_sk(), _dahai(0), {"type": "ryukyoku", "deltas": None}, END],
                                             [_sk(1), _dahai(1), _ryu([0, 0, 0, 0]), END]),
    "missing deltas in the last kyoku": _game([_sk(), _dahai(0), _ryu([0, 0, 0, 0]), END],
                                              [_sk(1), _dahai(1), {"type": "hora", "actor": 2, "target": 1}, END]),
    "missing deltas on the second of two rons": _game([_sk(3), _dahai(0), _hora(1, 0, [-8000, 8000, 0, 0]),
                                                      {"type": "hora", "actor": 3, "target": 0}, END]),
    "reach_accepted after the last hora": _game([_sk(), _dahai(0), _hora(1, 0, [-8000, 8000, 0, 0]),
                                                 {"type": "reach_accepted", "actor": 2}, END]),
    "no hora or ryukyoku after the last start_kyoku": _game([_sk(), _dahai(0), _ryu([3000, -1000, -1000, -1000]), END],
                                                            [_sk(1, (28000, 24000, 24000, 24000)), *_reach(1), END]),
    "no start_kyoku": _game(),
    "no start_kyoku, a ryukyoku without deltas": _game([_dahai(0), {"type": "ryukyoku"}, END]),
    "no start_kyoku, a hora with deltas": _game([_dahai(0), _hora(1, 0, [-1000, 1000, 0, 0]), END]),
}
ERRORS = {"missing deltas in the last kyoku": "NO_DELTAS", "missing deltas on the second of two rons": "NO_DELTAS",
          "no start_kyoku": "NO_KYOKU", "no start_kyoku, a ryukyoku without deltas": "NO_DELTAS",
          "no start_kyoku, a hora with deltas": "NO_KYOKU"}


@pytest.mark.parametrize("name", list(EDGE))
def test_edge_cases(name):
    status = _check([EDGE[name]])
    assert G.STATUS[int(status[0])] == ERRORS.get(name, "OK")


def test_round_winds_and_the_final_ranking():
    a = G.encode([EDGE["east, south, west and north rounds"], EDGE["a tie stays in seat order"],
                  EDGE["a total under 100000 tops up the leader"], EDGE["scores near the int32 limits"]])
    feat, rank, final, status = G.run_emul(a)
    assert not status.any()
    assert feat[:8, 0].tolist() == [0, 3, 4, 7, 8, 11, 8, 11]  # W and N rounds share 7 + kyoku (grp.rs:153-160)
    assert feat[:8, 1].tolist() == [0, 3] * 4 and feat[:8, 2].tolist() == [1, 1] * 4
    assert rank[1].tolist() == [0, 2, 1, 3] and final[1].tolist() == [30000, 20000, 30000, 20000]
    assert rank[2].tolist() == [0, 1, 2, 3] and final[2].tolist() == [31000, 30000, 20000, 19000]
    # 64-bit sums; the total (-4) is under 100000, so seat 0, first of the two leaders, takes the difference
    assert final[3].tolist() == [2 * 2147483647 + 100004, 2 * 2147483647, -2 * 2147483648, -2 * 2147483648]
    assert rank[3].tolist() == [0, 1, 2, 3]


def test_capacity_and_out_of_range_offsets(games):
    a = G.encode(games[:4])
    _, _, _, status = G.run_emul(a, n_hdr=int(a["ev_off"][3]) + 5)
    assert status[:3].tolist() == [0, 0, 0] and G.STATUS[int(status[3])] == "CAPACITY"
    _, _, _, status = G.run_emul(a, n_kyoku_words=int(a["ky_off"][2]) * 19)
    assert status[:2].tolist() == [0, 0] and {G.STATUS[int(s)] for s in status[2:]} == {"CAPACITY"}
    h = dict(a, ev_off=np.array([-1, 0, 0, 0], dtype=np.int32))
    assert G.STATUS[int(G.run_emul(h)[3][0])] == "CAPACITY"


# ---- the shared read helpers ---------------------------------------------------------------------------------------------------
def test_host_text_is_what_the_text_reader_returns(tmp_path):
    import gzip

    raw = b'{"a": 1}\r\n{"b": "\xc3\xa9"}\r\r\n\r{"c": 2}\n'
    p = tmp_path / "x.json.gz"
    with gzip.open(p, "wb") as f:
        f.write(raw)
    with gzip.open(p, "rt", encoding="utf-8") as f:
        want = f.read()
    assert _logio.read_gz(str(p)) == raw and _logio.host_text(raw) == want
    assert _logio.utf8_ok(raw) and not _logio.utf8_ok(b"\xff{}") and _logio.utf8_ok(b"{}")
    plain = tmp_path / "y.json"
    plain.write_bytes(raw)
    assert _logio.read_gz(str(plain)) is None and _logio.read_bytes(str(plain)) == raw  # every loader file is gunzipped


def test_augment_safety_counts_the_rewritten_fields():
    from mortal_b200.dataset import _augment_safe

    types = np.zeros(17, dtype=np.int64)
    types[dataset_codec.DAHAI] = 2
    assert _augment_safe(b'{"pai": "1m"} {"pai": "2m"}', types)
    assert not _augment_safe(b'{"pai": "1m"} {"pai": "2m"} {"type": "reach", "pai": 5}', types)
    assert not _augment_safe(b'{"type": "end_kyoku", "consumed": 1}', types)
    assert not _augment_safe(b'{"type": "ryukyoku", "ura_markers": 1}', types)
