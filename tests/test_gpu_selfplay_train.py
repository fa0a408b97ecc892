"""Self-play games handed to the trainer as device event words (mortal_b200/selfplay.py, csrc/mjx_selfplay.cuh) against the log path
over the same run's written files: decode_games against decode_dev, GameplayLoader.load_games against load_gz_log_files, and
SelfPlayDatasetsIter against FileDatasetsIter, for OneVsThree and TwoVsTwo arenas that write their logs and record their games in
one run. Everything must be equal bit for bit."""
import gzip
import json
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import reward_lib as R  # noqa: E402
from test_gpu_arena_logs import DevEngine  # noqa: E402

PTS = [90, 45, 0, -135]


def _play(tmp_path_factory, arena_cls, seed_count, tag):
    from mortal_b200 import _lib

    _lib.init(0)
    d = tmp_path_factory.mktemp(tag)
    arena = arena_cls(disable_progress_bar=True, log_dir=str(d))
    arena.record_games = True
    arena.py_vs_py(DevEngine(torch, "trainee", salt=0.3), DevEngine(torch, "baseline", salt=-0.2), (61000, 17), seed_count)
    return arena.last_games, list(arena.last_log_paths), arena.last_results


@pytest.fixture(scope="module")
def one_vs_three(tmp_path_factory):
    from mortal_b200.libriichi.arena import OneVsThree

    return _play(tmp_path_factory, OneVsThree, 4, "ovt")


@pytest.fixture(scope="module")
def two_vs_two(tmp_path_factory):
    from mortal_b200.libriichi.arena import TwoVsTwo

    return _play(tmp_path_factory, TwoVsTwo, 4, "tvt")


@pytest.fixture(scope="module")
def grp():
    return R.random_grp(64, 2, 21)


def _blobs(paths):
    out = []
    for p in paths:
        with gzip.open(p, "rb") as f:
            out.append(f.read())
    return out


def test_games_hold_the_run(one_vs_three, two_vs_two):
    for games, paths, res in (one_vs_three, two_vs_two):
        assert len(games) == len(paths) == res["ranks"].shape[0]
        assert (games.ranks == res["ranks"]).all() and (games.scores == res["scores"]).all()
        for g, p in enumerate(paths):  # the start_game line the writer wrote is the one load_games builds
            first = json.loads(_blobs([p])[0].split(b"\n", 1)[0])
            assert first == games.first_event(g)


@pytest.mark.parametrize("arena", ["one_vs_three", "two_vs_two"])
@pytest.mark.parametrize("augment", [False, True])
def test_decode_games_equals_decode_dev_of_the_files(request, arena, augment):
    from mortal_b200.selfplay import decode_games
    from mortal_b200.validate_logs import decode_dev

    games, paths, _ = request.getfixturevalue(arena)
    A = decode_games(games, augment=augment)
    B = decode_dev(_blobs(paths), 0, augment=augment, deltas=True)
    assert B.accept.all() and A.accept.all()
    np.testing.assert_array_equal(A.counts[:, :4], B.counts[:, :4])
    for k in ("ev_off", "ev_cnt", "ky_off", "hora_off"):
        np.testing.assert_array_equal(getattr(A, k), getattr(B, k))
    assert torch.equal(A.offs, B.offs)
    for k in ("hdr", "lines", "kyoku", "hora"):
        assert torch.equal(getattr(A, k), getattr(B, k)), k
    ty = B.hdr & 0xFF
    at = (ty == 12) | (ty == 13)  # hora, ryukyoku: the only entries of deltas / has_deltas either writes
    assert at.any() and torch.equal(A.has_deltas[at], B.has_deltas[at]) and torch.equal(A.deltas[at], B.deltas[at])
    assert not A.has_deltas[~at].any()


def test_decode_games_subset_and_errors(one_vs_three):
    from mortal_b200.selfplay import SelfPlayGames, decode_games
    from mortal_b200.validate_logs import decode_dev

    games, paths, _ = one_vs_three
    idx = [5, 0, 9]
    A = decode_games(games, idx)
    B = decode_dev(_blobs([paths[i] for i in idx]), 0, deltas=True)
    assert torch.equal(A.hdr, B.hdr) and torch.equal(A.kyoku, B.kyoku) and torch.equal(A.hora, B.hora)
    words = games.words.clone()
    words[2, 10] = 0  # not an event type (word 10: the event after the first start_kyoku and its 9 payload words)
    bad = SelfPlayGames(words, games.lens.clone(), games.log_cap, games.names, games.seeds, games.ranks, games.scores)
    with pytest.raises(RuntimeError, match=rf"game 2 \(seed {games.seeds[2][0]}, {games.seeds[2][1]}\): corrupt"):
        decode_games(bad, [1, 2])
    decode_games(bad, [1, 3])  # the other games still convert
    lens = games.lens.clone()
    lens[1] = games.log_cap + 5
    over = SelfPlayGames(games.words, lens, games.log_cap, games.names, games.seeds, games.ranks, games.scores)
    with pytest.raises(RuntimeError, match=rf"game 1 .*event log overflow: {games.log_cap + 5} words > capacity {games.log_cap}"):
        decode_games(over)


def _same_gameplays(a, b):
    assert len(a) == len(b)
    for ga, gb in zip(a, b):
        assert len(ga) == len(gb)
        for x, y in zip(ga, gb):
            assert x.take_player_id() == y.take_player_id() and x.player_name == y.player_name
            assert torch.equal(x.take_obs(), y.take_obs()) and torch.equal(x.take_masks().cpu(), y.take_masks().cpu())
            for k in ("take_actions", "take_at_kyoku", "take_dones", "take_apply_gamma", "take_at_turns", "take_shantens"):
                assert getattr(x, k)() == getattr(y, k)(), k
            gx, gy = x.take_grp(), y.take_grp()
            assert np.array_equal(gx.take_feature(), gy.take_feature())
            assert gx.take_rank_by_player() == gy.take_rank_by_player() and gx.take_final_scores() == gy.take_final_scores()


@pytest.mark.parametrize("version", [2, 3, 4])
@pytest.mark.parametrize("names", [["trainee"], None], ids=["trainee", "all"])
@pytest.mark.parametrize("augmented", [False, True])
def test_load_games_equals_load_gz_log_files(one_vs_three, two_vs_two, version, names, augmented):
    from mortal_b200.dataset import GameplayLoader

    for games, paths, _ in (one_vs_three, two_vs_two):
        loader = GameplayLoader(version, oracle=False, player_names=names, augmented=augmented)
        got = loader.load_games(games)
        want = loader.load_gz_log_files(paths)
        _same_gameplays(got, want)
        seats = sum(4 if names is None else g.count("trainee") for g in games.names)
        assert sum(len(g) for g in got) == seats and seats >= len(games)


@pytest.mark.parametrize("reserve_ratio,augmentation,augmented_first", [(0, False, False), (0.5, True, False), (0.5, True, True)])
def test_selfplay_iter_equals_file_iter(one_vs_three, grp, reserve_ratio, augmentation, augmented_first):
    from mortal_b200.dataloader import FileDatasetsIter
    from mortal_b200.selfplay import SelfPlayDatasetsIter

    games, paths, _ = one_vs_three
    kw = dict(file_batch_size=3, reserve_ratio=reserve_ratio, player_names=["trainee"], enable_augmentation=augmentation,
              augmented_first=augmented_first, grp=grp, batch_size=96)
    random.seed(1234)
    want = [tuple(t.clone() for t in b) for b in FileDatasetsIter(4, list(paths), PTS, **kw)]
    random.seed(1234)
    got = [tuple(t.clone() for t in b) for b in SelfPlayDatasetsIter(4, games, PTS, **kw)]
    assert len(got) == len(want) > 3
    for a, b in zip(got, want):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            assert x.dtype == y.dtype and x.device == y.device and torch.equal(x, y)


def test_record_games_without_log_dir_is_the_same_run(one_vs_three):
    from mortal_b200.libriichi.arena import OneVsThree

    games, _, _ = one_vs_three
    arena = OneVsThree(disable_progress_bar=True)
    arena.record_games = True
    arena.py_vs_py(DevEngine(torch, "trainee", salt=0.3), DevEngine(torch, "baseline", salt=-0.2), (61000, 17), 4)
    other = arena.last_games
    arena.record_games = False
    arena.py_vs_py(DevEngine(torch, "trainee", salt=0.3), DevEngine(torch, "baseline", salt=-0.2), (61000, 17), 1)
    assert arena.last_games is None  # a run without record_games does not leave the previous run's games
    assert torch.equal(other.lens, games.lens) and other.seeds == games.seeds and other.names == games.names
    for g in range(len(games)):
        n = int(games.lens[g])
        assert torch.equal(other.words[g, :n], games.words[g, :n])


def _train_cfg(tmp_path, games=8, repeats=2):
    from test_gpu_train import tiny_cfg

    cfg = tiny_cfg(tmp_path, "tp", tmp_path)
    cfg["baseline"]["train"] = dict(cfg["baseline"]["test"])
    cfg["train_play"] = {"default": {"games": games, "log_dir": str(tmp_path / "train_play"), "boltzmann_epsilon": 0.005,
                                     "boltzmann_temp": 0.05, "top_p": 1.0, "repeats": repeats}}
    return cfg


def _module_state(mods):
    return ([{k: v.clone() for k, v in m.state_dict().items()} for m in mods], [[x.training for x in m.modules()] for m in mods])


@pytest.mark.parametrize("freeze_bn", [False, True])
def test_train_player_sessions(tmp_path, monkeypatch, freeze_bn):
    from mortal_b200.model import DQN, Brain
    from mortal_b200.player import TrainPlayer

    monkeypatch.delenv("TRAIN_PLAY_PROFILE", raising=False)
    cfg = _train_cfg(tmp_path)
    dev = torch.device("cuda", 0)
    torch.manual_seed(3)
    mortal = Brain(conv_channels=32, num_blocks=2, version=4).to(dev)
    dqn = DQN(version=4).to(dev)
    mortal.freeze_bn(freeze_bn)
    mortal.train(); dqn.train()
    before = _module_state((mortal, dqn))
    player = TrainPlayer(cfg)
    seeds = []
    for session in range(3):
        seeds.append(player.train_seed)
        if session == 1:
            rankings, files = player.train_play(mortal, dqn, dev)
            assert len(files) == 8 and all(os.path.exists(f) for f in files)
        else:
            rankings, games = player.train_play_games(mortal, dqn, dev)
            assert len(games) == 8 and {n.count("trainee") for n in games.names} == {1}
            assert {s[1] for s in games.seeds} == {player.train_key}
            assert {s[0] for s in games.seeds} == set(range(seeds[-1], seeds[-1] + 2))
        assert rankings.sum() == 8 and rankings.shape == (4,)
        after = _module_state((mortal, dqn))
        for a, b in zip(before[0], after[0]):
            assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
        assert before[1] == after[1]
    assert seeds == [10000, 10000, 10002]  # repeats = 2: the seed advances by seed_count after every second session


# ---- train_online ---------------------------------------------------------------------------------------------------------------
STATE_KEYS = {"mortal", "current_dqn", "aux_net", "optimizer", "scheduler", "scaler", "steps", "timestamp", "best_perf", "config"}


def _online_cfg(tmp_path, name, min_q_weight=5.0):
    from test_gpu_train import tiny_cfg

    cfg = tiny_cfg(tmp_path, name, tmp_path)
    d = tmp_path / name
    cfg["control"].update(online=True, batch_size=64, save_every=2, test_every=4)
    cfg["cql"]["min_q_weight"] = min_q_weight
    cfg["baseline"]["train"] = dict(cfg["baseline"]["test"])
    cfg["train_play"] = {"default": {"games": 8, "log_dir": str(d / "train_play"), "boltzmann_epsilon": 0.005, "boltzmann_temp": 0.05,
                                     "top_p": 1.0, "repeats": 1}}
    cfg["online"] = {"history_window": 50, "enable_compile": False, "remote": {"host": "127.0.0.1", "port": 5000},
                     "server": {"buffer_dir": str(d / "buffer"), "drain_dir": str(d / "drain"), "capacity": 8,
                                "force_sequential": False}}
    return cfg


@pytest.fixture
def fixed_key(monkeypatch):
    import mortal_b200.player as player

    monkeypatch.setattr(player.secrets, "randbits", lambda n: 0x5EED)
    monkeypatch.delenv("TRAIN_PLAY_PROFILE", raising=False)


def test_train_online_rounds_save_test_play_and_resume(tmp_path, fixed_key, monkeypatch):
    import mortal_b200.selfplay as selfplay
    from mortal_b200.train import train_online

    sizes = []

    class Counting(selfplay.SelfPlayDatasetsIter):
        def build_iter(self):
            for b in super().build_iter():
                sizes.append(b[0].shape[0])
                yield b

    monkeypatch.setattr(selfplay, "SelfPlayDatasetsIter", Counting)
    cfg = _online_cfg(tmp_path, "run")
    _, _, _, opt, total = train_online(cfg, rounds=2)
    full = sum(1 for s in sizes if s == 64)
    assert total == full >= 4 and len(sizes) > full  # two rounds of trainee samples, the short tail batches skipped
    state = torch.load(cfg["control"]["state_file"], weights_only=True)
    assert set(state) == STATE_KEYS and state["config"]["control"]["online"] is True
    assert state["steps"] == total - total % 2
    assert os.path.exists(cfg["control"]["best_state_file"]) and os.path.isdir(cfg["test_play"]["log_dir"])
    assert not os.path.exists(cfg["train_play"]["default"]["log_dir"])  # no log is written
    sizes.clear()
    _, _, _, opt2, total2 = train_online(cfg, rounds=1)  # resumes the online state: optimizer and scheduler included
    assert total2 == state["steps"] + sum(1 for s in sizes if s == 64)
    assert opt2.state_dict()["state"] and len(opt2.state_dict()["state"]) == len(state["optimizer"]["state"])


def test_online_step_has_no_cql_term(tmp_path, one_vs_three, grp, monkeypatch):
    """the same initial weights and batches under two min_q_weight values: online, bit-equal parameters; offline (the control),
    different ones"""
    from mortal_b200.selfplay import SelfPlayDatasetsIter
    from mortal_b200.train import _Trainer

    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    games, _, _ = one_vs_three
    random.seed(5)
    batches = [tuple(t.clone() for t in b) for b in SelfPlayDatasetsIter(4, games, PTS, player_names=["trainee"], grp=grp,
                                                                          batch_size=64)][:3]
    assert all(b[0].shape[0] == 64 for b in batches)
    for online in (True, False):
        params = []
        for name, w in (("a", 5.0), ("b", 0.0)):
            cfg = _online_cfg(tmp_path, f"{name}{int(online)}", min_q_weight=w)
            cfg["control"]["save_every"] = cfg["control"]["test_every"] = 100  # no save or test play in between
            torch.manual_seed(7)
            T = _Trainer(cfg, online=online)
            for b in batches:
                T.step(*b)
            params.append([p.detach().clone() for m in (T.mortal, T.dqn, T.aux_net) for p in m.parameters()])
        same = all(torch.equal(x, y) for x, y in zip(*params))
        assert same == online, online


def test_train_online_from_offline_state_keeps_weights_and_starts_a_fresh_optimizer(tmp_path, fixed_key):
    from mortal_b200.model import mortal_state_dict
    from mortal_b200.train import train_online

    cfg = _online_cfg(tmp_path, "resume")
    train_online(cfg, rounds=1, steps=2)  # one save: an online state
    state = torch.load(cfg["control"]["state_file"], weights_only=True)
    state["config"]["control"]["online"] = False  # as if the offline trainer had written it
    state["steps"] = 40
    torch.save(state, cfg["control"]["state_file"])
    mortal, dqn, aux, opt, total = train_online(cfg, rounds=1, steps=0)
    assert total == 40 and not opt.state_dict()["state"]
    ref = mortal_state_dict(mortal)
    assert all(torch.equal(ref[k].cpu(), state["mortal"][k].cpu()) for k in ref)
    assert all(torch.equal(v, state["current_dqn"][k]) for k, v in dqn.state_dict().items())
    state["config"]["control"]["online"] = True
    torch.save(state, cfg["control"]["state_file"])
    _, _, _, opt, _ = train_online(cfg, rounds=1, steps=0)
    assert opt.state_dict()["state"]
