"""mortal/player.py:14-73 TestPlayer on the device: the trainee plays one-vs-three against a fixed baseline checkpoint in the
device arena, and the games' logs give its `Stat`.

The baseline is read from `[baseline.test] state_file` through `load_mortal` (any version, reference key layout) and runs as a
`DeviceEngine` with the rule-based agari guard, as the reference's MortalEngine does. The challenger is a `DeviceEngine` over the
live training modules; the engine plays a bf16 copy of them (`DeviceEngine.refresh`), so training resumes on untouched fp32
parameters and BatchNorm statistics.

mortal/player.py:75-157 TrainPlayer: the trainee (a `DeviceEngine` named `trainee` over the live modules, with the
`[train_play.<profile>]` exploration settings, profile from $TRAIN_PLAY_PROFILE, default `default`) plays one-vs-three against the
`[baseline.train]` checkpoint from seed (10000 + k * seed_count, train_key), the seed advancing every `repeats` sessions.
`train_play` writes the session's logs to the profile's `log_dir` as the reference does; `train_play_games` writes nothing and
returns the games as a `selfplay.SelfPlayGames` for `GameplayLoader.load_games`. Both leave the caller's modules in the training
mode they had, submodule by submodule (so frozen BatchNorms stay frozen): the engine puts them in eval mode while it plays.
"""
from __future__ import annotations

import logging
import os
import secrets
import shutil
from os import path

import numpy as np
import torch

from .dist import seed_block
from .engine import DeviceEngine
from .libriichi.arena import OneVsThree
from .model import load_mortal
from .stat import COUNTERS, Stat


class TestPlayer:
    def __init__(self, config):
        baseline_cfg = config["baseline"]["test"]
        device = torch.device(baseline_cfg["device"])
        state = torch.load(baseline_cfg["state_file"], weights_only=True, map_location=torch.device("cpu"))
        brain, dqn = load_mortal(state)
        self.baseline_engine = DeviceEngine(brain, dqn, version=brain.version, device=device, enable_amp=True,
                                            enable_rule_based_agari_guard=True, name="baseline")
        self.chal_version = config["control"]["version"]
        self.log_dir = path.abspath(config["test_play"]["log_dir"])
        self.cudnn_benchmark = config["control"].get("enable_cudnn_benchmark", False)

    def test_play(self, seed_count, mortal, dqn, device, group=None):
        """`seed_count` seeds x 4 games from seed (10000, 0x2000), the challenger in each seat once; logs in `log_dir` (emptied
        first); returns the challenger's Stat.

        With a torch.distributed `group` of several data-parallel ranks (all sharing `log_dir`'s file system), each rank plays its
        contiguous block of the seeds (dist.seed_block) on `device` and writes its games' logs under the names one process would
        give them; the Stat is the sum over the ranks of each rank's Stat of its own recorded games, the same on every rank."""
        import torch.distributed as dist

        world = dist.get_world_size(group) if group is not None else 1
        torch.backends.cudnn.benchmark = False
        engine_chal = DeviceEngine(mortal, dqn, version=self.chal_version, device=device, enable_amp=True, name="mortal")
        if world == 1:
            if path.isdir(self.log_dir):
                shutil.rmtree(self.log_dir)
            env = OneVsThree(disable_progress_bar=True, log_dir=self.log_dir, device=device.index or 0)
            env.py_vs_py(challenger=engine_chal, champion=self.baseline_engine, seed_start=(10000, 0x2000), seed_count=seed_count)
            stat = Stat.from_dir(self.log_dir, "mortal", disable_progress_bar=True)
        else:
            rank = dist.get_rank(group)
            if rank == 0 and path.isdir(self.log_dir):
                shutil.rmtree(self.log_dir)
            dist.barrier(group=group)
            start, count = seed_block(seed_count, rank, world)
            stat = Stat()
            if count:
                env = OneVsThree(disable_progress_bar=True, log_dir=self.log_dir, device=device.index or 0)
                env.record_games = True
                env.py_vs_py(challenger=engine_chal, champion=self.baseline_engine, seed_start=(10000 + start, 0x2000),
                             seed_count=count)
                stat = Stat.from_games(env.last_games, "mortal")
                env.last_games = None
            counters = torch.tensor([getattr(stat, c) for c in COUNTERS], dtype=torch.int64, device=device)
            dist.all_reduce(counters, group=group)
            stat = Stat(**dict(zip(COUNTERS, counters.tolist())))
        torch.backends.cudnn.benchmark = self.cudnn_benchmark
        return stat


class TrainPlayer:
    def __init__(self, config):
        baseline_cfg = config["baseline"]["train"]
        device = torch.device(baseline_cfg["device"])
        state = torch.load(baseline_cfg["state_file"], weights_only=True, map_location=torch.device("cpu"))
        brain, dqn = load_mortal(state)
        self.baseline_engine = DeviceEngine(brain, dqn, version=brain.version, device=device, enable_amp=True,
                                            enable_rule_based_agari_guard=True, name="baseline")
        profile = os.environ.get("TRAIN_PLAY_PROFILE", "default")
        logging.info(f"using profile {profile}")
        cfg = config["train_play"][profile]
        self.chal_version = config["control"]["version"]
        self.log_dir = path.abspath(cfg["log_dir"])
        self.train_key = secrets.randbits(64)
        self.train_seed = 10000
        self.seed_count = cfg["games"] // 4
        self.boltzmann_epsilon = cfg["boltzmann_epsilon"]
        self.boltzmann_temp = cfg["boltzmann_temp"]
        self.top_p = cfg["top_p"]
        self.repeats = cfg["repeats"]
        self.repeat_counter = 0
        self.cudnn_benchmark = config["control"].get("enable_cudnn_benchmark", False)

    def _play(self, mortal, dqn, device, log_dir):
        """one session -> (rankings, the arena); the seed advances after `repeats` sessions"""
        modes = [(m, m.training) for mod in (mortal, dqn) for m in mod.modules()]
        torch.backends.cudnn.benchmark = False
        try:
            engine_chal = DeviceEngine(mortal, dqn, version=self.chal_version, boltzmann_epsilon=self.boltzmann_epsilon,
                                       boltzmann_temp=self.boltzmann_temp, top_p=self.top_p, device=device, enable_amp=True,
                                       name="trainee")
            arena = OneVsThree(disable_progress_bar=True, log_dir=log_dir, device=device.index or 0)
            arena.record_games = log_dir is None
            rankings = arena.py_vs_py(challenger=engine_chal, champion=self.baseline_engine,
                                      seed_start=(self.train_seed, self.train_key), seed_count=self.seed_count)
        finally:
            for m, training in modes:
                m.training = training
            torch.backends.cudnn.benchmark = self.cudnn_benchmark
        self.repeat_counter += 1
        if self.repeat_counter == self.repeats:
            self.train_seed += self.seed_count
            self.repeat_counter = 0
        return np.array(rankings), arena

    def train_play(self, mortal, dqn, device):
        """one session with its logs in `log_dir` (emptied first) -> (rankings [4], the log files)"""
        if path.isdir(self.log_dir):
            shutil.rmtree(self.log_dir)
        rankings, _ = self._play(mortal, dqn, device, self.log_dir)
        return rankings, [path.join(self.log_dir, p) for p in os.listdir(self.log_dir)]

    def train_play_games(self, mortal, dqn, device):
        """one session, no files -> (rankings [4], selfplay.SelfPlayGames of its games)"""
        rankings, arena = self._play(mortal, dqn, device, None)
        return rankings, arena.last_games
