"""CPU checks of the online parameter server (mortal_b200/online.py Server), driven by scripted request sequences against the rules
of the reference's mortal/server.py, and of the `[online] actor_devices` config rejections, raised before any process exists."""
import multiprocessing
import threading

import pytest

from mortal_b200.online import Server


class _Games:
    """stands in for a selfplay.SelfPlayGames: the server only counts the games and reads their seeds"""

    def __init__(self, n, tag=0):
        self.seeds = [(tag, g) for g in range(n)]

    def __len__(self):
        return len(self.seeds)


def _recorder():
    events = []
    return events, lambda kind, **info: events.append((kind, info))


def test_overflow_comes_before_empty_param():
    s = Server(capacity=4, force_sequential=False)
    assert s.get_param(-1) == {"status": "empty param"}
    s.submit_replay(0, -1, _Games(4))
    assert s.get_param(-1) == {"status": "samples overflow"}  # no parameter was ever published: overflow still answers first
    s.submit_param("p1", is_idle=False)
    assert s.get_param(-1) == {"status": "samples overflow"}
    assert [x.param_version for x in s.drain()] == [-1]
    assert s.get_param(-1) == {"status": "ok", "snapshot": "p1", "param_version": 1}


def test_busy_only_under_force_sequential_and_cleared_by_an_idle_publish_only():
    for fs in (False, True):
        s = Server(capacity=8, force_sequential=fs)
        assert s.submit_param("idle", is_idle=True) == 1
        assert s.get_param(-1)["status"] == "ok"
        assert s.get_param(1)["status"] == ("trainer is busy" if fs else "ok")
        assert s.submit_param("train", is_idle=False) == 2
        res = s.get_param(1)
        assert res["status"] == ("trainer is busy" if fs else "ok")  # a non-idle publish does not clear it
        if not fs:
            assert res["snapshot"] == "train" and res["param_version"] == 2
        assert s.submit_param("idle2", is_idle=True) == 3
        assert s.get_param(1) == {"status": "ok", "snapshot": "idle2", "param_version": 3}
        assert s.get_param(3)["status"] == ("trainer is busy" if fs else "ok")
        assert s.idle_param_version == 3


def test_drain_empty_and_the_force_sequential_threshold():
    s = Server(capacity=8, force_sequential=False)
    assert s.drain() == []
    s.submit_replay(1, 3, _Games(4, 1))
    taken = s.drain()
    assert [(x.actor, x.param_version, len(x.games)) for x in taken] == [(1, 3, 4)]
    assert s.drain() == [] and s.buffer_size == 0

    s = Server(capacity=8, force_sequential=True)
    s.submit_replay(0, 1, _Games(4, 0))
    assert s.drain() == [] and s.buffer_size == 4  # below capacity: nothing moves
    s.submit_replay(1, 1, _Games(4, 1))
    taken = s.drain()
    assert [x.actor for x in taken] == [0, 1] and s.buffer_size == 0 and s.buffer == []
    s.submit_replay(0, 2, _Games(12, 0))  # above capacity: everything goes
    assert [len(x.games) for x in s.drain()] == [12]


def test_versions_are_monotone_and_events_are_in_order():
    events, monitor = _recorder()
    s = Server(capacity=4, force_sequential=False, monitor=monitor)
    versions = [s.submit_param(f"p{i}", is_idle=i % 3 == 0) for i in range(7)]
    assert versions == list(range(1, 8))
    assert s.idle_param_version == 7 and s.param_version == 7
    s.submit_replay(0, 7, _Games(4, 0))
    s.submit_replay(1, 6, _Games(4, 1))
    taken = s.drain()
    kinds = [k for k, _ in events]
    assert kinds == ["publish"] * 7 + ["submit", "submit", "drain"]
    assert [e["version"] for k, e in events if k == "publish"] == versions
    assert [e["is_idle"] for k, e in events if k == "publish"] == [i % 3 == 0 for i in range(7)]
    subs = [e for k, e in events if k == "submit"]
    assert [e["buffered"] for e in subs] == [4, 8] and subs[1]["seeds"] == [(1, g) for g in range(4)]
    drain = events[-1][1]
    assert drain["submissions"] == taken == [e["submission"] for e in subs] and drain["param_version"] == 7


def test_wait_param_and_drain_block_until_they_can_answer():
    s = Server(capacity=4, force_sequential=True)
    got = []
    t = threading.Thread(target=lambda: got.append(s.wait_param(-1)))
    t.start()
    t.join(0.2)
    assert t.is_alive()  # empty param: waiting
    s.submit_param("p", is_idle=True)
    t.join(5)
    assert not t.is_alive() and got[0]["param_version"] == 1

    t = threading.Thread(target=lambda: got.append(s.drain(wait=True)))
    t.start()
    s.submit_replay(0, 1, _Games(2))
    t.join(0.2)
    assert t.is_alive()  # 2 < capacity under force_sequential
    s.submit_replay(0, 1, _Games(2))
    t.join(5)
    assert not t.is_alive() and len(got[1]) == 2


def test_close_and_fail_wake_the_waiters():
    s = Server(capacity=4, force_sequential=True)
    got = []
    t = threading.Thread(target=lambda: got.append(s.wait_param(5)))
    t.start()
    s.close()
    t.join(5)
    assert got == [None]
    s.submit_replay(0, 1, _Games(4))
    assert s.buffer_size == 0  # a closed server takes no games

    s = Server(capacity=4, force_sequential=False)
    errors = []

    def drain():
        try:
            s.drain(wait=True)
        except RuntimeError as e:
            errors.append(str(e))

    t = threading.Thread(target=drain)
    t.start()
    s.fail("actor 1 (cuda:0) failed: boom")
    t.join(5)
    assert errors == ["actor 1 (cuda:0) failed: boom"]
    with pytest.raises(RuntimeError, match="actor 1"):
        s.submit_param("p", is_idle=False)


def _cfg(actor_devices, games=8, capacity=8, force_sequential=False):
    return {"control": {"version": 4, "online": True, "save_every": 2, "opt_step_every": 1, "test_every": 4},
            "resnet": {"conv_channels": 32, "num_blocks": 2},
            "train_play": {"default": {"games": games, "log_dir": "unused", "boltzmann_epsilon": 0.0, "boltzmann_temp": 0.05,
                                       "top_p": 1.0, "repeats": 1}},
            "online": {"history_window": 50, "actor_devices": actor_devices,
                       "server": {"capacity": capacity, "force_sequential": force_sequential}}}


def test_actor_device_config_rejections(monkeypatch):
    from mortal_b200.online import parse_actor_devices
    from mortal_b200.train import check_online_config, train_online

    monkeypatch.delenv("TRAIN_PLAY_PROFILE", raising=False)
    check_online_config(_cfg(["cuda:0", "cuda:0", "cuda:1"]))
    check_online_config(_cfg([]))  # empty: the sequential loop
    assert [str(d) for d in parse_actor_devices(["cuda", "cuda:3"])] == ["cuda:0", "cuda:3"]
    for bad in ("cpu", "meta", "cuda:x", 1):
        with pytest.raises(ValueError, match=r"actor_devices\[1\] = .* is not a CUDA device"):
            train_online(_cfg(["cuda:0", bad]))
    with pytest.raises(ValueError, match="must be a list"):
        train_online(_cfg("cuda:0"))
    check_online_config(_cfg(["cuda:0"], games=8, capacity=16))  # not sequential: any capacity is reached eventually
    check_online_config(_cfg(["cuda:0", "cuda:1"], games=8, capacity=16, force_sequential=True))
    with pytest.raises(ValueError, match=r"force_sequential = true with 1 actor\(s\) x 8 games per session = 8 games per round, "
                                         r"fewer than \[online.server\] capacity = 16"):
        train_online(_cfg(["cuda:0"], games=8, capacity=16, force_sequential=True))
    with pytest.raises(ValueError, match=r"2 actor\(s\) x 4 games per session = 8 games"):  # 7 games play one seed: 4
        train_online(_cfg(["cuda:0", "cuda:0"], games=7, capacity=9, force_sequential=True))
    assert multiprocessing.active_children() == []
