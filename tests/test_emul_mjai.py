"""The mjai decoder's logic (csrc/mjx_mjai.cuh, host build) against the host path: it accepts every well-formed log, in any
format Python's json reads the same way, with arrays identical to encode_log / encode_events; a hostile log is declined or decoded
identically."""
from collections import Counter

import numpy as np
import pytest

import log_mutations as LM
import mjai_lib as M
from validate_lib import emul_games


@pytest.fixture(scope="module")
def games():
    return emul_games(16, 1, seed0=223000) + emul_games(16, 0, seed0=224000)


def _check_accepted(texts, augment=False):
    blobs = [t.encode("utf-8") for t in texts]
    got = M.emul_decode(blobs, augment)
    for i, (b, g) in enumerate(zip(blobs, got)):
        want = M.host_decode(b, augment)
        assert want is not None, i
        assert g is not None, (i, b[:200])
        assert M.same(g, want), i


def test_golden_and_selfplay_logs(games):
    _check_accepted(M.golden_texts() + [M.game_text(g) for g in games])


def test_augment_matches_augment_events(games):
    _check_accepted(M.golden_texts()[:1] + [M.game_text(g) for g in games[:8]], augment=True)


def test_log_mutations_corpus(games):
    corpus = LM.mutated_corpus(games, 6, np.random.default_rng(3))
    blobs = [t.encode("utf-8") for _, t in corpus]
    got = M.emul_decode(blobs)
    for (cls, _), b, g in zip(corpus, blobs, got):
        want = M.host_decode(b)
        assert (g is None) == (want is None), cls  # every log the host encodes is accepted; every parse failure declined
        if g is not None:
            assert M.same(g, want), cls


def test_format_variations(games):
    rng = np.random.default_rng(17)
    texts = [M.vary(g, rng) for g in games for _ in range(3)] + [M.vary(g, rng) for g in [[{"type": "start_game"}]]]
    assert any("\r\n" in t for t in texts) and any("\\u" in t for t in texts) and any("名前" in t for t in texts)
    _check_accepted(texts)


def test_hostile_logs_are_declined_or_identical(games):
    rng = np.random.default_rng(29)
    base = [M.game_text(g) for g in games[:8]] + [M.vary(g, rng) for g in games[8:16]]
    corpus = M.hostile_corpus(base, 40, rng)
    got = M.emul_decode([b for _, b in corpus])
    declined = Counter()
    for (cls, b), g in zip(corpus, got):
        want = M.host_decode(b)
        if g is None:
            declined[cls] += 1
        else:
            assert want is not None and M.same(g, want), (cls, b[:300])
    # the classes Python always rejects are always declined (a '\r' may land before a '\n', a key may not be where the
    # duplicate goes: those classes also make logs Python reads unchanged)
    for cls in ("nan", "key_escape", "u2028", "control", "non_object", "trailing", "deep", "bad_utf8", "newline_run"):
        assert declined[cls] == 40, (cls, declined)


def test_edge_cases():
    sk = ('{"type":"start_kyoku","bakaze":"E","dora_marker":"1m","kyoku":1,"honba":0,"kyotaku":0,"oya":0,'
          '"scores":[25000,25000,25000,25000],"tehais":[' + ",".join(['["1m","1m","1m","1m","2m","2m","2m","2m","3m","3m","3m","3m","?"]'] * 4) + "]}")
    cases = {
        b"": False, b"\n\n  \t\n": False, b'{"type":"end_game"}': True, b'{"type":"end_game"}\r': False,
        b'{"type":"end_game"}\r\n\r\n': True, b'{"type":"end_game"}\x0c\n': False, b'\xef\xbb\xbf{"type":"end_game"}\n': False,
        b'{"type":"reach","actor":-0}\n': True, b'{"type":"reach","actor":3}\n': True, b'{"type":"reach","actor":1.0}\n': False,
        b'{"type":"reach","actor":true}\n': False, b'{"type":"dahai","actor":0,"pai":"5mr","tsumogiri":false}\n': True,
        b'{"type":"dahai","actor":0,"pai":"5mr","tsumogiri":0}\n': False, b'{"type":"hora","actor":0,"target":1,"deltas":null}\n': True,
        b'{"type":"hora","actor":0,"target":1,"ura_markers":["1m","2m","3m","4m","5m","6m"],"deltas":[-1,2,3,4]}\n': True,
        b'{"type":"hora","actor":0,"target":1,"deltas":[1,2,3]}\n': False, b'{"type":"ryukyoku","deltas":[0,0,0,2147483648]}\n': False,
        b'{"type":"ryukyoku","deltas":{"a":1}, "x": [1,]}\n': False, b'{"type":"end_kyoku","meta":{"a":[1e400,-0.0]}}\n': True,
        sk.encode() + b"\n": True, sk.replace('"E"', '"P"').encode(): False, sk.replace('"kyoku":1', '"kyoku":5').encode(): False,
        b'{"type":"ankan","actor":0,"consumed":["?","?","?","?"]}\n': True, b'{"type":"chi","actor":0,"target":3,"pai":"?","consumed":["?","?"]}': True,
        b'{"type":"tsumo","actor":0,"pai":"0m"}': False, b'{"type":"dora","dora_marker":"5sr"} ': True,
        # a decline followed by runs of line breaks longer than the 64-entry queue of line ends
        b"x" + b"\n" * 127: False, b"not json\n" + b"\n" * 200 + b'{"type":"end_game"}\n': False,
        b'{"type":"end_game"}' + b"\n" * 300 + b'{"type":"end_game"}' + b"\r\n" * 70: True,
    }
    got = M.emul_decode(list(cases))
    for (b, accept), g in zip(cases.items(), got):
        assert (g is not None) == accept, b
        want = M.host_decode(b)
        if g is not None:
            assert want is not None and M.same(g, want), b
