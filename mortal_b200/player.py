"""mortal/player.py:14-73 TestPlayer on the device: the trainee plays one-vs-three against a fixed baseline checkpoint in the
device arena, and the games' logs give its `Stat`.

The baseline is read from `[baseline.test] state_file` through `load_mortal` (any version, reference key layout) and runs as a
`DeviceEngine` with the rule-based agari guard, as the reference's MortalEngine does. The challenger is a `DeviceEngine` over the
live training modules; the engine plays a bf16 copy of them (`DeviceEngine.refresh`), so training resumes on untouched fp32
parameters and BatchNorm statistics. (TrainPlayer, which feeds online training, is not built: online training is not supported.)
"""
from __future__ import annotations

import shutil
from os import path

import torch

from .engine import DeviceEngine
from .libriichi.arena import OneVsThree
from .model import load_mortal
from .stat import Stat


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

    def test_play(self, seed_count, mortal, dqn, device):
        """`seed_count` seeds x 4 games from seed (10000, 0x2000), the challenger in each seat once; logs in `log_dir` (emptied
        first); returns the challenger's Stat"""
        torch.backends.cudnn.benchmark = False
        engine_chal = DeviceEngine(mortal, dqn, version=self.chal_version, device=device, enable_amp=True, name="mortal")
        if path.isdir(self.log_dir):
            shutil.rmtree(self.log_dir)
        env = OneVsThree(disable_progress_bar=True, log_dir=self.log_dir, device=device.index or 0)
        env.py_vs_py(challenger=engine_chal, champion=self.baseline_engine, seed_start=(10000, 0x2000), seed_count=seed_count)
        stat = Stat.from_dir(self.log_dir, "mortal", disable_progress_bar=True)
        torch.backends.cudnn.benchmark = self.cudnn_benchmark
        return stat
