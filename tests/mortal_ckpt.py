"""Mortal checkpoints for the tests, rebuilt from a key list: the cases pinned by tests/golden/mortal_model_outputs.npz
(tools/extract_model_fixtures.py runs the reference's own Brain / DQN on them) and the deterministic weight rule both sides use.

A checkpoint here is what mortal/train.py saves: {'mortal': Brain.state_dict(), 'current_dqn': DQN.state_dict(), 'config': ...}
with the reference's key names. Every tensor is a function of (case seed, key index) only, so a state dict is regenerated from the
fixture's ordered (key, shape) lists instead of being stored."""
from __future__ import annotations

import json
import os

import numpy as np

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mortal_model_outputs.npz")
CONV_CHANNELS, NUM_BLOCKS, ROWS = 32, 2, 6
# name: (version, is_oracle, seed)
CASES = {"v1": (1, False, 101), "v2": (2, False, 102), "v3": (3, False, 103), "v4": (4, False, 104),
         "v1_oracle": (1, True, 105), "v4_oracle": (4, True, 106)}


def tensor_for(seed: int, index: int, key: str, shape, keys) -> np.ndarray:
    """The value of key number `index` of a state dict whose keys are `keys`: BatchNorm statistics and affines away from the
    identity (running_var 0.5..1.5, running_mean N(0, 0.1), weight 0.5..1.5, bias N(0, 0.1)); weights N(0, 1 / fan_in); other
    biases N(0, 0.1); num_batches_tracked 0."""
    rng = np.random.default_rng([seed, index])
    prefix, leaf = key.rsplit(".", 1)
    shape = tuple(shape)
    if leaf == "num_batches_tracked":
        return np.zeros(shape, dtype=np.int64)
    bn = prefix + ".running_var" in keys
    if leaf == "running_var" or (bn and leaf == "weight"):
        return rng.uniform(0.5, 1.5, shape).astype(np.float32)
    if leaf in ("running_mean", "bias"):
        return rng.normal(0.0, 0.1, shape).astype(np.float32)
    fan_in = int(np.prod(shape[1:]))
    return rng.normal(0.0, 1.0 / np.sqrt(fan_in), shape).astype(np.float32)


def state_dict(seed: int, key_shapes) -> dict:
    import torch

    keys = {k for k, _ in key_shapes}
    return {k: torch.from_numpy(tensor_for(seed, i, k, s, keys)) for i, (k, s) in enumerate(key_shapes)}


def config(version: int) -> dict:
    """mortal's config.toml as a checkpoint carries it; version 1 leaves control.version out (player.py's default)"""
    control = {} if version == 1 else {"version": version}
    return {"control": control, "resnet": {"conv_channels": CONV_CHANNELS, "num_blocks": NUM_BLOCKS}}


def observations(version: int, is_oracle: bool, seed: int):
    """a seeded batch: 0/1 observations (10 % ones), invisible observations for oracle cases, legal masks with at least one action"""
    from mortal_b200.model import OBS_ROWS, ORACLE_ROWS

    rng = np.random.default_rng([seed, 1 << 20])
    obs = (rng.random((ROWS, OBS_ROWS[version], 34)) < 0.1).astype(np.float32)
    inv = (rng.random((ROWS, ORACLE_ROWS[version], 34)) < 0.1).astype(np.float32) if is_oracle else None
    masks = rng.random((ROWS, 46)) < 0.3
    masks[:, 45] = True
    return obs, inv, masks


def load_fixture():
    """{case: dict(brain_keys, dqn_keys, outputs...)} from the golden file"""
    z = np.load(FIXTURE)
    out = {}
    for name in CASES:
        d = {"brain_keys": json.loads(str(z[f"{name}/brain_keys"])), "dqn_keys": json.loads(str(z[f"{name}/dqn_keys"]))}
        for k in ("phi", "mu", "logsig", "q", "obs", "inv", "masks"):
            if f"{name}/{k}" in z:
                d[k] = z[f"{name}/{k}"]
        out[name] = d
    return out


def checkpoint(name: str, fx: dict) -> dict:
    version, _, seed = CASES[name]
    return {"mortal": state_dict(seed, fx["brain_keys"]), "current_dqn": state_dict(seed + 1000, fx["dqn_keys"]), "config": config(version)}
