"""The validation kernel's logic (csrc/mjx_validate.cuh, single-lane host build) against the oracle's restatement of
bin/validate_logs.rs, over self-play logs of the emulated environment and every mutation class of tests/log_mutations.py."""
import json
from collections import Counter

import numpy as np
import pytest

import log_mutations as LM
from validate_lib import emul_games, emul_validate, oracle_validate


@pytest.fixture(scope="module")
def games():
    return emul_games(32, 1, seed0=123000) + emul_games(32, 0, seed0=124000)


def test_selfplay_logs_are_valid(games):
    texts = ["\n".join(json.dumps(e) for e in g) + "\n" for g in games]
    assert emul_validate(texts) == [None] * len(texts)
    assert [oracle_validate(t) for t in texts] == [None] * len(texts)


def test_mutations_match_the_oracle(games):
    corpus = LM.mutated_corpus(games, 12, np.random.default_rng(7))
    got = emul_validate([t for _, t in corpus])
    want = [oracle_validate(t) for _, t in corpus]
    assert got == want
    failed = Counter(c for (c, _), v in zip(corpus, want) if v is not None)
    assert set(failed) == set(LM.CLASSES), failed  # every class produces failures
    assert all(v.status != "UNSUPPORTED" for v in got if v is not None)  # the capacity guard is never reached
