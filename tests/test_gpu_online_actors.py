"""train_online with self-play actors (`[online] actor_devices`, mortal_b200/online.py) on the GPU, on the tiny config of
test_gpu_selfplay_train with greedy self-play (boltzmann_epsilon = 0) and fixed actor keys, so every session can be played again:
one force_sequential actor against the sequential loop (same games, bit-identical final state), two overlapped actors against the
parameter server's rules, an actor error, and an actor on a second GPU. No test leaves a process behind."""
import itertools
import multiprocessing
import random
import secrets

import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from test_gpu_selfplay_train import _online_cfg  # noqa: E402


@pytest.fixture(autouse=True)
def no_process_left(monkeypatch):
    monkeypatch.delenv("TRAIN_PLAY_PROFILE", raising=False)
    yield
    assert multiprocessing.active_children() == []


def _cfg(tmp_path, name, actor_devices, force_sequential, capacity=8, submit_every=100):
    cfg = _online_cfg(tmp_path, name)
    cfg["train_play"]["default"]["boltzmann_epsilon"] = 0.0
    cfg["control"]["submit_every"] = submit_every
    cfg["online"]["server"].update(capacity=capacity, force_sequential=force_sequential)
    if actor_devices is not None:
        cfg["online"]["actor_devices"] = actor_devices
    return cfg


class _Events:
    """a train_online monitor: every event in order, with a clone of every published snapshot"""

    def __init__(self):
        self.events, self.snapshots = [], {}

    def __call__(self, kind, **info):
        if kind == "publish":
            self.snapshots[info["version"]] = {m: {k: v.clone() for k, v in sd.items()} for m, sd in info["snapshot"].items()}
        self.events.append((kind, info))

    def of(self, kind):
        return [info for k, info in self.events if k == kind]


def _game_rows(games):
    return [(games.seeds[g], int(games.lens[g]), games.words[g, :int(games.lens[g])].cpu()) for g in range(len(games))]


def _same_rows(a, b):
    assert len(a) == len(b)
    for (sa, la, wa), (sb, lb, wb) in zip(a, b):
        assert sa == sb and la == lb and torch.equal(wa, wb)


def test_one_sequential_actor_equals_the_sequential_loop(tmp_path, monkeypatch):
    import mortal_b200.player as player
    from mortal_b200.train import train_online

    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(secrets, "randbits", lambda n: 0x5EED)  # the sequential TrainPlayer's key and the actor's
    seq_games = []
    play = player.TrainPlayer.train_play_games

    def recording(self, *a):
        rankings, games = play(self, *a)
        seq_games.append(games)
        return rankings, games

    monkeypatch.setattr(player.TrainPlayer, "train_play_games", recording)
    runs = {}
    for name, devices in (("seq", None), ("act", ["cuda:0"])):
        cfg = _cfg(tmp_path, name, devices, force_sequential=True)
        events = _Events()
        random.seed(1234)
        torch.manual_seed(7)
        total = train_online(cfg, rounds=2, monitor=events)[4]
        runs[name] = (cfg, events, total)
    (seq_cfg, _, seq_total), (act_cfg, events, act_total) = runs["seq"], runs["act"]

    assert len(seq_games) == 2
    drains = events.of("drain")
    assert len(drains) == 2 and [len(d["submissions"]) for d in drains] == [1, 1]
    for sg, d in zip(seq_games, drains):
        _same_rows(_game_rows(d["submissions"][0].games), _game_rows(sg))
    # the second session played the parameters of the first pass's idle publish, as the sequential loop plays them
    idle = [p["version"] for p in events.of("publish") if p["is_idle"]]
    assert [d["submissions"][0].param_version for d in drains] == idle[:2]

    assert act_total == seq_total > 0
    a = torch.load(act_cfg["control"]["state_file"], weights_only=True)
    b = torch.load(seq_cfg["control"]["state_file"], weights_only=True)
    assert a["steps"] == b["steps"]
    for key in ("mortal", "current_dqn", "aux_net"):
        assert a[key].keys() == b[key].keys() and all(torch.equal(a[key][k], b[key][k]) for k in a[key]), key
    oa, ob = a["optimizer"], b["optimizer"]
    assert oa["param_groups"] == ob["param_groups"] and oa["state"].keys() == ob["state"].keys()
    for i in oa["state"]:
        assert all(torch.equal(oa["state"][i][k], ob["state"][i][k]) for k in oa["state"][i])
    assert a["scheduler"] == b["scheduler"]


def test_two_overlapped_actors_follow_the_server_rules(tmp_path, monkeypatch):
    from mortal_b200.model import DQN, Brain
    from mortal_b200.player import TrainPlayer
    from mortal_b200.train import train_online

    keys = itertools.count(0x1000)
    monkeypatch.setattr(secrets, "randbits", lambda n: next(keys))
    cfg = _cfg(tmp_path, "two", ["cuda:0", "cuda:0"], force_sequential=False, capacity=8, submit_every=1)
    events = _Events()
    total = train_online(cfg, rounds=3, monitor=events)[4]
    assert total > 0

    pending, published, n_drains = [], 0, 0
    games_per_session = cfg["train_play"]["default"]["games"]
    for kind, info in events.events:
        if kind == "publish":
            assert info["version"] == published + 1
            published = info["version"]
        elif kind == "submit":
            assert 1 <= info["param_version"] <= published  # never a version before it was published
            assert info["buffered"] <= cfg["online"]["server"]["capacity"] + 2 * games_per_session - 1
            pending.append(info["submission"])
        else:
            assert info["submissions"] == pending  # exactly the submissions since the previous drain, in order
            pending = []
            n_drains += 1
    assert n_drains == 3
    subs = [s for d in events.of("drain") for s in d["submissions"]]
    assert all({k for _, k in s.games.seeds} == {0x1000 + s.actor} for s in subs)  # one key per actor, drawn in this process

    # a submission played again in this process, from the snapshot of its version and its seeds
    sub = subs[-1]
    snap = events.snapshots[sub.param_version]
    dev = torch.device("cuda", 0)
    mortal = Brain(version=4, **cfg["resnet"]).to(dev).eval()
    dqn = DQN(version=4).to(dev)
    mortal.load_state_dict(snap["mortal"])
    dqn.load_state_dict(snap["dqn"])
    p = TrainPlayer(cfg)
    p.train_seed, p.train_key = sub.games.seeds[0]
    rankings, games = p.train_play_games(mortal, dqn, dev)
    _same_rows(_game_rows(games), _game_rows(sub.games))
    assert (games.ranks == sub.games.ranks).all()


def test_an_actor_error_names_the_actor_and_stops_the_others(tmp_path):
    from mortal_b200.train import train_online

    cfg = _cfg(tmp_path, "err", ["cuda:0", "cuda:0"], force_sequential=False)
    cfg["baseline"]["train"]["state_file"] = str(tmp_path / "missing.pth")
    with pytest.raises(RuntimeError, match=r"actor [01] \(cuda:0\) failed:(.|\n)*missing\.pth"):
        train_online(cfg, rounds=1)


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_an_actor_on_another_gpu(tmp_path, monkeypatch):
    from mortal_b200.train import train_online

    monkeypatch.setattr(secrets, "randbits", lambda n: 0x77)
    cfg = _cfg(tmp_path, "gpu1", ["cuda:1"], force_sequential=True)
    events = _Events()
    total = train_online(cfg, rounds=1, monitor=events)[4]
    (drain,) = events.of("drain")
    (sub,) = drain["submissions"]
    assert total > 0 and len(sub.games) == 8 and sub.games.words.device == torch.device("cuda", 0)
    assert {s[1] for s in sub.games.seeds} == {0x77}
