"""Arena mjai logs rendered on the device (mortal_b200/mjai_write.py, csrc/mjx_mjai_write.cuh) against the host writer
(mortal_b200/mjai_log.write_logs): the same seeds through both paths must give the same file names in the same order and the same
decompressed bytes. Engines are deterministic (Q is a function of the observation and the mask) and the arena's clock is replaced by
a counter, so eval_time_ns is reproducible."""
import gzip
import os
import types

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch

    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from mortal_b200 import _lib

    _lib.init(0)
    return torch


def _q_of(torch, obs, masks, salt):
    w = torch.linspace(-1.0, 1.0 + salt, obs.shape[-1], device=obs.device, dtype=torch.float32)
    q = (obs[:, : 46, :].float() * w).sum(-1) + 0.37 * obs[:, 46:92, :].float().sum(-1) + salt
    return q.masked_fill(~masks, -float("inf"))


class DevEngine:
    engine_type = "mortal"
    is_oracle = False
    enable_quick_eval = True
    enable_rule_based_agari_guard = False

    def __init__(self, torch, name, version=4, salt=0.0, guard=False, oracle=False):
        self.torch, self.name, self.version, self.salt = torch, name, version, salt
        self.enable_rule_based_agari_guard, self.is_oracle = guard, oracle

    def react_device(self, obs, masks, invisible_obs=None):
        q = _q_of(self.torch, obs, masks, self.salt)
        if invisible_obs is not None:
            q = q + 0.01 * invisible_obs[:, :46, :].float().sum(-1).masked_fill(~masks, 0)
        return q.argmax(-1), q


class HostEngine:
    """the reference protocol (react_batch over lists of numpy arrays) with per-row is_greedy flags"""
    engine_type = "mortal"
    is_oracle = False
    enable_quick_eval = True
    enable_rule_based_agari_guard = False

    def __init__(self, torch, name, version=4, salt=0.0):
        self.torch, self.name, self.version, self.salt = torch, name, version, salt

    def react_batch(self, obs, masks, invisible_obs):
        t = self.torch
        o, m = t.as_tensor(np.stack(obs)), t.as_tensor(np.stack(masks))
        q = _q_of(t, o, m, self.salt)
        a = q.argmax(-1)
        greedy = (o[:, :8, :].sum((1, 2)).long() % 3 != 0)  # a function of the observation
        return a.tolist(), q.tolist(), m.tolist(), greedy.tolist()


def _run(torch, monkeypatch, tmp, cls, chal, champ, seed, count, host, **opts):
    from mortal_b200.libriichi import arena as A

    clock = iter(range(10 ** 6, 10 ** 12, 1237))
    monkeypatch.setattr(A, "time", types.SimpleNamespace(perf_counter_ns=lambda: next(clock)))
    d = os.path.join(tmp, "host" if host else "dev")
    ar = cls(disable_progress_bar=True, log_dir=d)
    ar.host_log_writer = host
    for k, v in opts.items():
        setattr(ar, k, v)
    torch.manual_seed(0)
    ar.py_vs_py(chal, champ, seed, count)
    monkeypatch.undo()
    return ar


def _same(torch, monkeypatch, tmp_path, cls, chal, champ, seed, count, **opts):
    dev = _run(torch, monkeypatch, str(tmp_path), cls, chal, champ, seed, count, False, **opts)
    host = _run(torch, monkeypatch, str(tmp_path), cls, chal, champ, seed, count, True, **opts)
    assert [os.path.basename(p) for p in dev.last_log_paths] == [os.path.basename(p) for p in host.last_log_paths]
    assert dev.last_meta_error is None and host.last_meta_error is None
    assert dev.last_log_timing and not host.last_log_timing  # the device writer ran on one and only on one
    metas = kans = 0
    for a, b in zip(dev.last_log_paths, host.last_log_paths):
        x, y = gzip.open(a).read(), gzip.open(b).read()
        assert x == y, (a, _first_diff(x, y))
        metas += x.count(b'"meta"')
        kans += x.count(b'"kan_select"')
    return len(dev.last_log_paths), metas, kans


def _first_diff(a, b):
    for i, (x, y) in enumerate(zip(a.split(b"\n"), b.split(b"\n"))):
        if x != y:
            k = next(j for j in range(min(len(x), len(y)) + 1) if j == min(len(x), len(y)) or x[j] != y[j])
            return f"line {i}, byte {k}:\n  device {x[max(0, k - 300):k + 200]!r}\n  host   {y[max(0, k - 300):k + 200]!r}"
    return "line counts differ"


def test_one_engine_for_every_seat(torch, monkeypatch, tmp_path):
    from mortal_b200.libriichi.arena import OneVsThree

    e = DevEngine(torch, "solo")
    n, metas, _ = _same(torch, monkeypatch, tmp_path, OneVsThree, e, e, (7100, 3), 4)
    assert n == 16 and metas > 16 * 100


def test_challenger_and_champion(torch, monkeypatch, tmp_path):
    from mortal_b200.libriichi.arena import OneVsThree

    _same(torch, monkeypatch, tmp_path, OneVsThree, DevEngine(torch, "chal", salt=0.5), DevEngine(torch, "champ"), (7200, 5), 4)


def test_host_protocol_pipeline_with_greedy_flags(torch, monkeypatch, tmp_path):
    from mortal_b200.libriichi.arena import OneVsThree

    n, metas, _ = _same(torch, monkeypatch, tmp_path, OneVsThree, HostEngine(torch, "h1", salt=0.25), HostEngine(torch, "h2"),
                        (7300, 1), 4)
    assert n == 16 and metas > 0


def test_mixed_versions_guard_oracle_fast_forward(torch, monkeypatch, tmp_path):
    from mortal_b200.libriichi.arena import OneVsThree

    _same(torch, monkeypatch, tmp_path, OneVsThree, DevEngine(torch, "v3", version=3, guard=True),
          DevEngine(torch, "v4", oracle=True), (7400, 9), 3)
    _same(torch, monkeypatch, tmp_path / "ff", OneVsThree, DevEngine(torch, "a"), DevEngine(torch, "b"), (7450, 9), 3,
          fast_forward_steps=40)


def test_without_meta_and_two_vs_two(torch, monkeypatch, tmp_path):
    from mortal_b200.libriichi.arena import OneVsThree, TwoVsTwo

    _, metas, _ = _same(torch, monkeypatch, tmp_path, OneVsThree, DevEngine(torch, "a"), DevEngine(torch, "b"), (7500, 2), 2,
                        log_meta=False)
    assert metas == 0
    n, _, _ = _same(torch, monkeypatch, tmp_path / "tvt", TwoVsTwo, DevEngine(torch, "x"), DevEngine(torch, "y", salt=1.0), (7600, 2), 6)
    assert n == 12


def test_1024_games_with_kan_select(torch, monkeypatch, tmp_path):
    from mortal_b200.libriichi.arena import OneVsThree

    n, metas, kans = _same(torch, monkeypatch, tmp_path, OneVsThree, DevEngine(torch, "a", salt=0.1), DevEngine(torch, "b"),
                           (8000, 11), 256)
    assert n == 1024 and kans > 0 and metas > 1024 * 100
