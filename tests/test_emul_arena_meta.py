"""The arena's host-protocol loop (pinned host buffers, two parts) on the emulated environment, logged through the host writer: every
logged dahai's meta is the decision that produced that discard. Until the recorder got a copy of each cycle's actions, it kept views
of the reused action buffer, so every cycle's meta was paired with the last cycle's actions."""
import gzip
import json

import numpy as np
import torch

from emul_batch_env import EmulBatchEnv
from mortal_b200 import mjai_log
from mortal_b200.libriichi.arena import OneVsThree


class LoggedEmulEnv(EmulBatchEnv):
    def enable_log(self):
        self._e.enable_log()

    @property
    def log_len(self):
        return torch.from_numpy(self._e.log_lens())

    def read_log(self):
        return self._e.read_log()


class RandomQ:
    """the reference protocol; Q a pseudo-random function of the observation, the action its legal argmax"""
    engine_type = "mortal"
    version = 4
    is_oracle = False
    enable_quick_eval = True
    enable_rule_based_agari_guard = False

    def __init__(self, name):
        self.name = name

    def react_batch(self, obs, masks, invisible_obs):
        o, m = np.stack(obs), np.stack(masks).astype(bool)
        w = np.random.default_rng(5).standard_normal((o.shape[1] * o.shape[2], 46)).astype(np.float32)
        q = o.reshape(len(o), -1) @ w + np.arange(46, dtype=np.float32) * 1e-3
        q = np.where(m, q, -np.inf).astype(np.float32)
        return q.argmax(1).tolist(), q.tolist(), m.tolist(), [True] * len(o)


def test_host_protocol_meta_is_the_decision_that_made_the_event(tmp_path):
    arena = OneVsThree(disable_progress_bar=True, log_dir=str(tmp_path))
    arena.env_factory = LoggedEmulEnv
    arena.py_vs_py(RandomQ("a"), RandomQ("b"), (6100, 4), 2)  # two seeds: two parts stepped alternately
    assert arena.last_meta_error is None
    checked = calls = 0
    for path in arena.last_log_paths:
        for ev in (json.loads(ln) for ln in gzip.open(path, "rt")):
            m = ev.get("meta")
            if m is None or ev["type"] not in mjai_log.AGENT_EVENT_ACTIONS:
                continue
            legal = [a for a in range(46) if (m["mask_bits"] >> a) & 1]
            chosen = legal[int(np.argmax(m["q_values"]))]  # the engine's decision on the row the meta came from
            assert chosen in mjai_log.AGENT_EVENT_ACTIONS[ev["type"]], (path, ev)  # the meta's row made this event type
            if ev["type"] == "dahai":
                assert mjai_log.TILE_NAMES[chosen] == ev["pai"], (path, ev)
            checked += 1
            calls += ev["type"] in ("chi", "pon", "daiminkan", "reach")
    assert checked > 8 * 100 and calls > 8
