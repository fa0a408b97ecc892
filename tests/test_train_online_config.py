"""CPU checks of train_online's config rejections (mortal_b200/train.py): each is raised before anything touches the device, and
train() keeps rejecting `online = true` with a pointer to train_online."""
import pytest


def _cfg(games=8, capacity=8, profile="default", **control):
    return {"control": {"version": 4, "online": True, "save_every": 2, "opt_step_every": 1, "test_every": 4, **control},
            "resnet": {"conv_channels": 32, "num_blocks": 2},
            "train_play": {profile: {"games": games, "log_dir": "unused", "boltzmann_epsilon": 0.005, "boltzmann_temp": 0.05,
                                     "top_p": 1.0, "repeats": 1}},
            "online": {"history_window": 50, "server": {"capacity": capacity}}}


def test_online_config_rejections(monkeypatch):
    from mortal_b200.train import check_online_config, train, train_online

    monkeypatch.delenv("TRAIN_PLAY_PROFILE", raising=False)
    check_online_config(_cfg())
    with pytest.raises(ValueError, match="train_online"):
        train(_cfg())
    with pytest.raises(ValueError, match="version 1"):
        train_online(_cfg(version=1))
    with pytest.raises(ValueError, match="games must be at least 4"):
        train_online(_cfg(games=3))
    with pytest.raises(ValueError, match="capacity must be at least 1"):
        train_online(_cfg(capacity=0))
    with pytest.raises(ValueError, match=r"no \[train_play.default\] profile"):
        train_online(_cfg(profile="other"))
    monkeypatch.setenv("TRAIN_PLAY_PROFILE", "other")
    check_online_config(_cfg(profile="other"))
    with pytest.raises(ValueError, match=r"no \[train_play.other\] profile"):
        train_online(_cfg())
    bad = _cfg()
    bad["control"]["test_every"] = 3
    with pytest.raises(ValueError, match="test_every a multiple of save_every"):
        train_online(bad)
