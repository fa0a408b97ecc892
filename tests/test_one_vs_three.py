"""mortal_b200.one_vs_three and Stat.from_games on the host: the [1v3] config rules (the reference's seed schedule, the drawn key,
what is rejected before any model is loaded), Stat.from_games over emulated self-play games against Stat.from_dir over the same
run's written logs and against the host build of k_arena_words + k_stat_logs, and the driver end to end on the emulated arena
with two stub engines."""
import io
import json
import re

import numpy as np
import pytest

import stat_lib as S
import test_emul_selfplay as SP
from mortal_b200 import one_vs_three as ovt
from mortal_b200.libriichi.arena import AKOCHAN_UNSUPPORTED, OneVsThree
from mortal_b200.stat import COUNTERS, Stat, _host_log_stat
from test_emul_arena_meta import LoggedEmulEnv


def _config(**over):
    side = lambda name: {"device": "cuda:0", "name": name, "state_file": f"/nonexistent/{name}.pth", "stochastic_latent": False,
                         "enable_compile": False, "enable_amp": True, "enable_rule_based_agari_guard": True}
    cfg = {"seed_key": 7, "games_per_iter": 8, "iters": 3, "log_dir": "", "challenger": side("mortal"),
           "champion": side("baseline"), "akochan": {"enabled": False, "dir": "", "tactics": ""}}
    cfg.update(over)
    return {"1v3": cfg}


def _counters(st):
    return {c: getattr(st, c) for c in COUNTERS}


# ---- config ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("games_per_iter,iters", [(2000, 500), (8, 3), (7, 2), (4, 1), (4, 0)])
def test_seed_schedule_is_the_references(games_per_iter, iters):
    P = ovt.plan(_config(games_per_iter=games_per_iter, iters=iters))
    spi = games_per_iter // 4
    assert P.seeds_per_iter == spi
    assert P.seeds == list(range(10000, 10000 + spi * iters, spi))
    assert ovt.plan(_config(games_per_iter=games_per_iter, iters=iters), iters=2).seeds == [10000, 10000 + spi]


def test_seed_key():
    P = ovt.plan(_config(seed_key=0x2000))
    assert (P.key, P.key_drawn) == (0x2000, False)
    drawn = [ovt.plan(_config(seed_key=-1)) for _ in range(3)]
    cfg = _config()
    del cfg["1v3"]["seed_key"]
    drawn.append(ovt.plan(cfg))  # an absent key is drawn too
    assert all(p.key_drawn and 0 <= p.key < 1 << 64 for p in drawn)
    assert len({p.key for p in drawn}) == len(drawn)


def test_log_dir_and_iters_per_call():
    assert ovt.plan(_config(log_dir="")).log_dir is None
    cfg = _config()
    del cfg["1v3"]["log_dir"]
    assert ovt.plan(cfg).log_dir is None
    assert ovt.plan(_config(log_dir="/x/1v3")).log_dir == "/x/1v3"
    assert ovt.plan(_config()).iters_per_call == 1 and ovt.plan(_config(iters_per_call=4)).iters_per_call == 4
    for bad in (0, -1, 1.5):
        with pytest.raises(ValueError, match="iters_per_call"):
            ovt.plan(_config(iters_per_call=bad))


def _rejects(monkeypatch, config, exc, match):
    """one_vs_three(config) raises exc before any engine is loaded or any game is played"""
    def fail(*a, **k):
        raise AssertionError("nothing may be loaded or played")

    monkeypatch.setattr(ovt, "load_engine", fail)
    monkeypatch.setattr(ovt, "OneVsThree", fail)
    out = io.StringIO()
    with pytest.raises(exc, match=match):
        ovt.one_vs_three(config, out=out)
    assert out.getvalue() == ""


def test_rejected_before_anything_is_loaded(monkeypatch):
    ako = _config(akochan={"enabled": True, "dir": "/a", "tactics": "/t.json"})
    _rejects(monkeypatch, ako, NotImplementedError, re.escape(AKOCHAN_UNSUPPORTED))
    with pytest.raises(NotImplementedError) as arena_exc:
        OneVsThree().ako_vs_py()
    assert str(arena_exc.value) == AKOCHAN_UNSUPPORTED
    for g in (0, 3):
        _rejects(monkeypatch, _config(games_per_iter=g), ValueError, "0 seeds")
    cfg = _config()
    cfg["1v3"]["champion"]["device"] = "cuda:1"
    _rejects(monkeypatch, cfg, ValueError, "differ")
    cfg = _config()
    cfg["1v3"]["challenger"]["device"] = cfg["1v3"]["champion"]["device"] = "cpu"
    _rejects(monkeypatch, cfg, ValueError, "CUDA device")
    cfg = _config()
    cfg["1v3"]["champion"]["name"] = "mortal"
    _rejects(monkeypatch, cfg, ValueError, "both named")
    cfg = _config()
    cfg["1v3"]["champion"]["device"] = "cuda"  # the current device, 0 in a fresh process: the same as cuda:0
    assert ovt.plan(cfg).device == 0


# ---- Stat.from_games on the host path ---------------------------------------------------------------------------------------
class Stub:
    """the reference protocol, deterministic and cheap: the highest legal action id, or the lowest one with low=True (version 1
    observations, the cheapest to encode on the emulated environment)"""
    engine_type = "mortal"
    version = 1
    is_oracle = False
    enable_quick_eval = True
    enable_rule_based_agari_guard = False

    def __init__(self, name, low=False):
        self.name, self.low = name, low

    def react_batch(self, obs, masks, invisible_obs):
        m = np.stack(masks).astype(bool)
        a = m.argmax(1) if self.low else 45 - m[:, ::-1].argmax(1)
        q = np.where(m, np.arange(46, dtype=np.float32) * (-1.0 if self.low else 1.0), -np.inf)
        return a.tolist(), q.tolist(), m.tolist(), [True] * len(a)


class EmulOneVsThree(OneVsThree):
    """the arena on the host-emulated environment"""

    def __init__(self, **kw):
        super().__init__(**kw)
        self.env_factory = LoggedEmulEnv


@pytest.fixture(scope="module")
def session(tmp_path_factory):
    d = tmp_path_factory.mktemp("ovt_logs")
    arena = EmulOneVsThree(disable_progress_bar=True, log_dir=str(d))
    arena.record_games = True
    arena.py_vs_py(Stub("mortal"), Stub("baseline", low=True), (10000, 0x2000), 3)
    return arena.last_games, list(arena.last_log_paths), str(d)


def test_from_games_equals_from_dir(session):
    games, paths, d = session
    assert len(games) == len(paths) == 12 and games.words.device.type == "cpu"
    for name, seats in (("mortal", 1), ("baseline", 3)):
        got = Stat.from_games(games, name)
        assert _counters(got) == _counters(Stat.from_dir(d, name)), name
        assert got.game == seats * len(games)
    assert _counters(Stat.from_games(games, "nobody")) == _counters(Stat())
    idx = [1, 4, 5, 11]
    for name in ("mortal", "baseline"):
        want = sum((_host_log_stat(paths[g], name) for g in idx), Stat())
        assert _counters(Stat.from_games(games, name, idx)) == _counters(want)
    assert _counters(Stat.from_games(games, "mortal", [])) == _counters(Stat())


def test_from_games_equals_the_emulated_kernels(session):
    """the host build of k_arena_words (count + fill) and of k_stat_logs over its arrays give from_games's counters"""
    games, _, _ = session
    words = games.words.numpy().view(np.uint64)
    lens = games.lens.numpy()
    counts, per_game = SP.convert(words, lens)
    assert (counts[:, 0] == SP.OK).all()
    hdr, ky, dl, hs = [], [], [], []
    ev_off, ev_cnt, ky_off = (np.zeros(len(games), dtype=np.int32) for _ in range(3))
    ne = nk = 0
    for g, a in enumerate(per_game):
        ev_off[g], ev_cnt[g], ky_off[g] = ne, len(a["hdr"]), nk
        ne += len(a["hdr"]); nk += len(a["kyoku"])
        hdr.append(a["hdr"]); ky.append(a["kyoku"].reshape(-1)); dl.append(a["deltas"]); hs.append(a["has"])
    arrays = dict(hdr=np.ascontiguousarray(np.concatenate(hdr)), ev_off=ev_off, ev_cnt=ev_cnt,
                  kyoku=np.ascontiguousarray(np.concatenate(ky)), ky_off=ky_off,
                  deltas=np.ascontiguousarray(np.concatenate(dl), dtype=np.int32), has=np.ascontiguousarray(np.concatenate(hs)))
    for name in ("mortal", "baseline"):
        masks = [sum(1 << s for s, n in enumerate(games.names[g]) if n == name) for g in range(len(games))]
        out, status = S.run_emul(arrays, masks)
        assert (status == 0).all()
        got = dict(zip(S.NAMES, (int(x) for x in out.sum(0))))
        assert got == _counters(Stat.from_games(games, name)), name


def test_from_games_corrupt_and_overflowed_words(session):
    from mortal_b200.selfplay import SelfPlayGames

    games, _, _ = session

    def copy(words, lens):
        return SelfPlayGames(words, lens, games.log_cap, games.names, games.seeds, games.ranks, games.scores)

    words = games.words.clone()
    words[2, 0] = 0xFF  # not an event type
    g2 = games.seeds[2]
    with pytest.raises(RuntimeError, match=rf"self-play game 2 \(seed {g2[0]}, {g2[1]}\): corrupt event log"):
        Stat.from_games(copy(words, games.lens), "mortal")
    assert Stat.from_games(copy(words, games.lens), "mortal", [0, 1, 3]).game == 3  # the other games are unaffected
    lens = games.lens.clone()
    lens[5] = games.log_cap + 1
    g5 = games.seeds[5]
    with pytest.raises(RuntimeError, match=rf"self-play game 5 \(seed {g5[0]}, {g5[1]}\): event log overflow"):
        Stat.from_games(copy(games.words, lens), "baseline")


# ---- the driver on the emulated arena ------------------------------------------------------------------------------------
LINE = re.compile(r"challenger rankings: \[(\d+) (\d+) (\d+) (\d+)\] \((\S+), (\S+)pt\)")


@pytest.fixture()
def emulated(monkeypatch):
    engines = {"mortal": Stub("mortal"), "baseline": Stub("baseline", low=True)}
    monkeypatch.setattr(ovt, "load_engine", lambda section, device: engines[section["name"]])
    monkeypatch.setattr(ovt, "OneVsThree", EmulOneVsThree)
    return engines


def _reference_lines(rankings):
    """what mortal/one_vs_three.py prints for these per-iteration rankings"""
    lines = []
    for i, r in enumerate(rankings):
        r = np.array([int(x) for x in r])
        avg_rank = r @ np.arange(1, 5) / r.sum()
        avg_pt = r @ np.array([90, 45, 0, -135]) / r.sum()
        lines += ["-" * 50, f"# {i}", f"challenger rankings: {r} ({avg_rank}, {avg_pt}pt)"]
    return lines


def test_driver_prints_the_references_lines(emulated, tmp_path):
    cfg = _config(games_per_iter=8, iters=2, seed_key=0x2000, log_dir=str(tmp_path / "logs"))
    out = io.StringIO()
    res = ovt.one_vs_three(cfg, out=out)
    text = out.getvalue().splitlines()
    assert text[:6] == _reference_lines(res.rankings)
    assert all(LINE.fullmatch(text[k]) for k in (2, 5))
    assert res.rankings.shape == (2, 4) and (res.rankings.sum(1) == 8).all()
    assert res.seeds == [10000, 10002] and res.key == 0x2000
    # the rankings of every iteration are those of a direct py_vs_py on its seeds
    for i, seed in enumerate(res.seeds):
        arena = EmulOneVsThree(disable_progress_bar=True)
        assert arena.py_vs_py(emulated["mortal"], emulated["baseline"], (seed, 0x2000), 2) == res.rankings[i].tolist()
    # the written logs are the reference's files, and both Stats are from_dir over them
    names = sorted(p.name for p in (tmp_path / "logs").iterdir())
    assert names == sorted(f"{s}_{0x2000}_{c}.json.gz" for s in range(10000, 10004) for c in "abcd")
    for name, st in (("mortal", res.challenger), ("baseline", res.champion)):
        assert _counters(st) == _counters(Stat.from_dir(str(tmp_path / "logs"), name))
    assert res.challenger.game == 16 and res.champion.game == 48
    assert res.challenger.total_pt(ovt.PTS) / 16 == pytest.approx(res.avg_pt)
    # the report: both sides' Stat reports under their headers, then the average rank pt with its standard error
    rest = "\n".join(text[6:])
    assert rest == res.report()
    assert f"challenger mortal (x1)\n{res.challenger.reference_text()}\n\n" in rest
    assert f"champion baseline (x3)\n{res.champion.reference_text()}\n\n" in rest
    se = np.std(res.set_pts, ddof=1) / np.sqrt(4)
    assert rest.endswith(f"challenger avg rank pt {res.avg_pt:.6f} ± {se:.6f} (standard error over 4 duplicate sets of 4 games)")


def test_iters_per_call_prints_the_same_lines(emulated, tmp_path):
    outs, results = [], []
    for k in (1, 2, 3):
        out = io.StringIO()
        log_dir = tmp_path / f"logs{k}"
        results.append(ovt.one_vs_three(_config(games_per_iter=4, iters=3, iters_per_call=k, log_dir=str(log_dir)), out=out))
        outs.append(out.getvalue())
        assert sorted(p.name for p in log_dir.iterdir()) == sorted(f"{s}_7_{c}.json.gz" for s in range(10000, 10003) for c in "abcd")
    assert outs[0] == outs[1] == outs[2]
    assert outs[0].splitlines()[:9] == _reference_lines(results[0].rankings)
    for r in results[1:]:
        assert (r.rankings == results[0].rankings).all() and (r.set_pts == results[0].set_pts).all()


def test_cli_summary_round_trips(emulated, tmp_path, capsys):
    cfg = tmp_path / "config.toml"
    cfg.write_text(
        "[1v3]\nseed_key = 4660\ngames_per_iter = 4\niters = 2\nlog_dir = ''\n"
        + "".join(f"[1v3.{side}]\ndevice = 'cuda:0'\nname = '{name}'\nstate_file = '/nonexistent'\nstochastic_latent = false\n"
                  f"enable_compile = false\nenable_amp = true\nenable_rule_based_agari_guard = true\n"
                  for side, name in (("challenger", "mortal"), ("champion", "baseline")))
        + "[1v3.akochan]\nenabled = false\ndir = ''\ntactics = ''\n")
    summary = tmp_path / "summary.json"
    assert ovt.main([str(cfg), "--summary", str(summary)]) == 0
    printed = capsys.readouterr().out
    s = json.loads(summary.read_text())
    assert s["seed_key"] == 4660 and s["seeds_per_iter"] == 1 and s["seeds"] == [10000, 10001]
    assert printed.splitlines()[:6] == _reference_lines(s["rankings"])
    assert s["challenger"]["name"] == "mortal" and s["challenger"]["seats"] == 1
    assert s["champion"]["name"] == "baseline" and s["champion"]["seats"] == 3
    chal, cham = Stat(**s["challenger"]["counters"]), Stat(**s["champion"]["counters"])
    assert chal.game == 8 and cham.game == 24
    assert f"challenger mortal (x1)\n{chal.reference_text()}\n" in printed
    assert f"champion baseline (x3)\n{cham.reference_text()}\n" in printed
    assert s["avg_pt"] == pytest.approx(chal.total_pt(ovt.PTS) / 8)
