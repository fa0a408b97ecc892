"""k_validate_logs on the GPU: arena logs are valid, mutated logs get the oracle's verdict, verdicts do not depend on batch
order or batching, hostile word sequences get a verdict without a failed call, and the CLI names exactly the bad files."""
import gzip
import json
import os
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest

import log_mutations as LM
from validate_lib import oracle_validate

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Eng:
    engine_type, version, is_oracle, enable_quick_eval, enable_rule_based_agari_guard, name = "mortal", 4, False, True, False, "e"

    def react_device(self, obs, masks):
        q = torch.rand(masks.shape, device=masks.device)
        q[:, :34] += 2.0 * obs[:, 876, :] + obs[:, 875, :]
        q = q.masked_fill(~masks, -1.0)
        return q.argmax(-1), q


@pytest.fixture(scope="module")
def arena_logs(tmp_path_factory):
    from mortal_b200.libriichi.arena import OneVsThree

    d = tmp_path_factory.mktemp("arena")
    OneVsThree(disable_progress_bar=True, log_dir=str(d)).py_vs_py(_Eng(), _Eng(), (77000, 11), 256)  # 4 games per seed
    files = sorted(os.path.join(d, f) for f in os.listdir(d))
    return {f: gzip.open(f, "rt").read() for f in files}


def test_arena_logs_are_valid(arena_logs):
    from mortal_b200.validate_logs import validate_logs

    assert len(arena_logs) == 1024
    assert any('"meta"' in t for t in arena_logs.values())  # the decision meta of Mortal's logs is ignored
    assert validate_logs(list(arena_logs.values())) == [None] * 1024


@pytest.fixture(scope="module")
def mutated(arena_logs):
    games = [[json.loads(x) for x in t.splitlines()] for t in list(arena_logs.values())[:256]]
    corpus = LM.mutated_corpus(games, 370, np.random.default_rng(2024))
    return corpus, [oracle_validate(t) for _, t in corpus]


def test_mutated_logs_match_the_oracle(mutated):
    from mortal_b200.validate_logs import validate_logs

    corpus, want = mutated
    assert len(corpus) >= 4000
    got = validate_logs([t for _, t in corpus])
    bad = [(c, g, w) for (c, _), g, w in zip(corpus, got, want) if g != w]
    assert not bad, bad[:5]
    failed = Counter(c for (c, _), w in zip(corpus, want) if w is not None)
    assert all(failed[c] >= 50 for c in LM.CLASSES), failed
    assert all(v.status != "UNSUPPORTED" for v in got if v is not None)  # the capacity guard is never reached


def test_order_and_batching_do_not_change_verdicts(mutated):
    from mortal_b200.validate_logs import validate_logs

    corpus, want = mutated
    texts = [t for _, t in corpus]
    perm = np.random.default_rng(5).permutation(len(texts))
    shuffled = validate_logs([texts[i] for i in perm])
    assert [shuffled[int(np.where(perm == i)[0][0])] for i in range(len(texts))] == want
    parts = []
    for lo, hi in ((0, 1), (1, 700), (700, 2001), (2001, len(texts))):
        parts += validate_logs(texts[lo:hi])
    assert parts == want


def test_malformed_words_get_a_verdict(arena_logs):
    from mortal_b200.validate_logs import encode_log, run_packed

    enc = [encode_log(t) for t in list(arena_logs.values())[:64]]
    rows = run_packed(LM.malformed_batch(enc, 2000, np.random.default_rng(12)))
    assert rows.shape == (2000, 4)
    assert ((rows[:, 0] >= 0) & (rows[:, 0] <= 4)).all()
    assert (rows[:, 0] != 0).sum() > 1000  # hostile input is rejected, not replayed


def test_cli_names_the_bad_files(arena_logs, tmp_path):
    texts = list(arena_logs.values())[:6]
    events = [json.loads(x) for x in texts[0].splitlines()]
    for seed in range(50):  # a riichi inserted at random: keep the first one the oracle rejects as not tenpai
        bad_text = LM.mutate(events, "riichi_not_tenpai", np.random.default_rng(seed))
        if oracle_validate(bad_text) is not None and oracle_validate(bad_text).reason == "can_riichi":
            break
    (tmp_path / "a" / "b").mkdir(parents=True)
    layout = {"a/ok1.json": texts[1], "a/b/ok2.json.gz": texts[2], "ok3.json.gz": texts[3], "a/b/bad.json.gz": bad_text,
              "a/bad2.json": "{\"type\": \"start_game\"}\nnot json\n", "ignored.txt": "garbage"}
    for name, text in layout.items():
        p = tmp_path / name
        if name.endswith(".gz"):
            with gzip.open(p, "wt") as f:
                f.write(text)
        else:
            p.write_text(text)
    r = subprocess.run([sys.executable, "-m", "mortal_b200.validate_logs", str(tmp_path)], cwd=ROOT, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr
    named = [ln.split("error in log ", 1)[1] for ln in r.stdout.splitlines() if ln.startswith("error in log ")]
    assert named == [str(tmp_path / "a" / "b" / "bad.json.gz"), str(tmp_path / "a" / "bad2.json")]
    line = oracle_validate(bad_text).line
    assert f"fails can_riichi at line {line}" in r.stdout
    assert "fails to parse (json) at line 2" in r.stdout
