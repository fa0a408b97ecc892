"""Stat.from_games and the 1v3 evaluation (mortal_b200.one_vs_three) on the GPU: from_games over a session's device words equals
Stat.from_dir over the same session's written logs, counter for counter, for the challenger (one seat per game), the champion
(three seats), a subset of the games and games forced through the host fallback; the CLI with two small checkpoints in the
reference's layout gives the rankings of direct py_vs_py calls on the same seeds, the reference's file names, the stat CLI's
report for each side, the same output for the same seed_key, and a summary that round-trips."""
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from test_gpu_arena_logs import DevEngine  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _counters(st):
    from mortal_b200.stat import COUNTERS

    return {c: getattr(st, c) for c in COUNTERS}


@pytest.fixture(scope="module")
def session(tmp_path_factory):
    from mortal_b200 import _lib
    from mortal_b200.libriichi.arena import OneVsThree

    _lib.init(0)
    d = tmp_path_factory.mktemp("ovt_session")
    arena = OneVsThree(disable_progress_bar=True, log_dir=str(d))
    arena.record_games = True
    arena.py_vs_py(DevEngine(torch, "mortal", salt=0.3), DevEngine(torch, "baseline", salt=-0.2), (10000, 0x2000), 16)
    games = arena.last_games
    assert games.words.is_cuda and len(games) == 64
    return games, list(arena.last_log_paths), str(d)


def test_from_games_equals_from_dir(session):
    from mortal_b200.stat import Stat

    games, paths, d = session
    for name, seats in (("mortal", 1), ("baseline", 3)):
        got = Stat.from_games(games, name)
        assert _counters(got) == _counters(Stat.from_dir(d, name)), name
        assert got.game == seats * len(games)


def test_from_games_subset(session, tmp_path):
    from mortal_b200.stat import Stat

    games, paths, _ = session
    idx = [3, 0, 17, 18, 40, 63]
    for g in idx:
        shutil.copy(paths[g], tmp_path)
    for name in ("mortal", "baseline"):
        assert _counters(Stat.from_games(games, name, idx)) == _counters(Stat.from_dir(str(tmp_path), name)), name


def test_from_games_host_fallback(session, monkeypatch):
    """games whose kernel status is non-zero (their deltas hidden from k_stat_logs, so it reports NO_DELTAS) are counted on the
    host with the same result; games on the host are counted there entirely"""
    from mortal_b200 import stat
    from mortal_b200.selfplay import SelfPlayGames
    from mortal_b200.stat import Stat

    games, paths, d = session
    forced = {5, 22}
    statuses = []
    real = stat._stat_logs_dev

    def hide_deltas(L, D, seats, dev, names):
        for j in forced:
            D.has_deltas[int(D.ev_off[j]):int(D.ev_off[j] + D.ev_cnt[j])] = 0
        sums, status = real(L, D, seats, dev, names)
        statuses.append(status.copy())
        return sums, status

    monkeypatch.setattr(stat, "_stat_logs_dev", hide_deltas)
    for name in ("mortal", "baseline"):
        assert _counters(Stat.from_games(games, name)) == _counters(Stat.from_dir(d, name)), name
    for status in statuses:
        assert set(np.nonzero(status)[0]) == forced
    monkeypatch.undo()
    on_host = SelfPlayGames(games.words.cpu(), games.lens.cpu(), games.log_cap, games.names, games.seeds, games.ranks, games.scores)
    for name in ("mortal", "baseline"):
        assert _counters(Stat.from_games(on_host, name, range(0, 64, 3))) == _counters(Stat.from_games(games, name, range(0, 64, 3)))


def test_from_games_corrupt_words_raise(session):
    from mortal_b200.selfplay import SelfPlayGames
    from mortal_b200.stat import Stat

    games, _, _ = session
    words = games.words.clone()
    words[7, 0] = 0xFF
    bad = SelfPlayGames(words, games.lens, games.log_cap, games.names, games.seeds, games.ranks, games.scores)
    s = games.seeds[7]
    with pytest.raises(RuntimeError, match=rf"self-play game 7 \(seed {s[0]}, {s[1]}\)"):
        Stat.from_games(bad, "mortal")


# ---- the CLI -----------------------------------------------------------------------------------------------------------------
def _write_config(path, ckpt, log_dir, key, iters_per_call=1):
    sides = "".join(f"[1v3.{side}]\ndevice = 'cuda:0'\nname = '{name}'\nstate_file = '{ckpt[name]}'\nstochastic_latent = false\n"
                    "enable_compile = false\nenable_amp = true\nenable_rule_based_agari_guard = true\n"
                    for side, name in (("challenger", "mortal"), ("champion", "baseline")))
    path.write_text(f"[1v3]\nseed_key = {key}\ngames_per_iter = 8\niters = 2\nlog_dir = '{log_dir}'\n"
                    f"iters_per_call = {iters_per_call}\n" + sides + "[1v3.akochan]\nenabled = false\ndir = ''\ntactics = ''\n")


def test_cli(tmp_path):
    import io

    import mortal_ckpt
    from mortal_b200 import one_vs_three as ovt
    from mortal_b200.libriichi.arena import OneVsThree
    from mortal_b200.stat import Stat
    from mortal_b200.train_grp import load_config

    fx = mortal_ckpt.load_fixture()
    ckpt = {"mortal": tmp_path / "v2.pth", "baseline": tmp_path / "v4.pth"}
    torch.save(mortal_ckpt.checkpoint("v2", fx["v2"]), ckpt["mortal"])
    torch.save(mortal_ckpt.checkpoint("v4", fx["v4"]), ckpt["baseline"])
    key = 0x1234
    logs = tmp_path / "logs"
    cfg = tmp_path / "config.toml"
    _write_config(cfg, ckpt, logs, key)
    summary = tmp_path / "summary.json"
    env = dict(os.environ, PYTHONPATH=ROOT)
    run = lambda *args: subprocess.run([sys.executable, "-m", *args], capture_output=True, text=True, cwd=ROOT, env=env, timeout=900)
    cli = run("mortal_b200.one_vs_three", str(cfg), "--summary", str(summary))
    assert cli.returncode == 0, cli.stderr
    lines = cli.stdout.splitlines()
    s = json.loads(summary.read_text())
    assert s["seed_key"] == key and s["seeds"] == [10000, 10002] and s["seeds_per_iter"] == 2
    # the reference's lines, and each iteration's rankings are those of a direct py_vs_py on its seeds
    config = load_config(str(cfg))
    chal, cham = ovt.load_engine(config["1v3"]["challenger"], 0), ovt.load_engine(config["1v3"]["champion"], 0)
    for i, seed in enumerate(s["seeds"]):
        direct = OneVsThree(disable_progress_bar=True).py_vs_py(challenger=chal, champion=cham, seed_start=(seed, key), seed_count=2)
        assert s["rankings"][i] == direct
        r = np.array(direct)
        avg_rank, avg_pt = r @ np.arange(1, 5) / r.sum(), r @ np.array([90, 45, 0, -135]) / r.sum()
        assert lines[3 * i:3 * i + 3] == ["-" * 50, f"# {i}", f"challenger rankings: {r} ({avg_rank}, {avg_pt}pt)"]
    # the log files are the reference's, and each side's report block is the stat CLI's report over them
    assert sorted(p.name for p in logs.iterdir()) == sorted(f"{sd}_{key}_{c}.json.gz" for sd in range(10000, 10004) for c in "abcd")
    for role, name, seats in (("challenger", "mortal", 1), ("champion", "baseline", 3)):
        st = run("mortal_b200.stat", str(logs), name)
        assert st.returncode == 0, st.stderr
        assert f"{role} {name} (x{seats})\n{st.stdout}" in cli.stdout + "\n"
        counters = Stat(**s[role]["counters"])
        assert st.stdout == counters.reference_text() + "\n"
        assert s[role]["name"] == name and s[role]["seats"] == seats and counters.game == 16 * seats
    # the same seed_key again (in this process, without logs): the same output
    config["1v3"]["log_dir"] = ""
    out = io.StringIO()
    res = ovt.one_vs_three(config, out=out)
    assert out.getvalue() == cli.stdout
    assert res.rankings.tolist() == s["rankings"] and res.avg_pt == pytest.approx(s["avg_pt"])
