"""The policy-net trainer on the device (mortal_b200.train, Brain.forward_train, train_ops.dqn_losses): the fused training step
against the torch path (Brain.forward + DQN + AuxNet + mortal/train.py's loss expressions) on the same batches and initial
weights -- first-step gradients of every parameter tensor against a float64 run, 20 AdamW steps of losses, BatchNorm running
statistics, frozen BatchNorm -- and train() on arena logs generated here: the state file's keys, strict loads through
load_mortal, play in DeviceEngine, resume, test play with the best-state copy, the illegal-action error and the command line."""
from __future__ import annotations

import copy
import os
import subprocess
import sys

import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import torch.nn.functional as F  # noqa: E402

from test_gpu_gameplay_decode import _Eng  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def models(version, c, n, seed):
    from mortal_b200.model import DQN, AuxNet, Brain

    torch.manual_seed(seed)
    brain, dqn, aux = Brain(conv_channels=c, num_blocks=n, version=version).cuda(), DQN(version=version).cuda(), AuxNet((4,)).cuda()
    with torch.no_grad():
        for m in brain.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.uniform_(0.7, 1.3)
                m.bias.normal_(0, 0.1)
    return brain, dqn, aux


def batch(version, b, seed, jitter=False):
    """a device batch of 0 / 1 observations. jitter=True adds U(0, 0.01) to them: identical tile columns of a 0 / 1 observation
    give exactly tied maxima in the gate's pooling, and amax's gradient jumps between tied entries, so a tie that rounding makes
    in one precision and not in another moves a gradient by far more than the rounding error a precision test measures"""
    from mortal_b200.model import OBS_ROWS

    g = torch.Generator(device="cuda").manual_seed(seed)
    obs = (torch.rand((b, OBS_ROWS[version], 34), generator=g, device="cuda") < 0.1).float()
    if jitter:
        obs += 0.01 * torch.rand(obs.shape, generator=g, device="cuda")
    masks = torch.rand((b, 46), generator=g, device="cuda") < 0.3
    masks[torch.arange(b, device="cuda"), torch.randint(0, 46, (b,), generator=g, device="cuda")] = True
    actions = torch.multinomial(masks.float(), 1, generator=g).squeeze(1)
    steps_to_done = torch.randint(0, 200, (b,), generator=g, device="cuda")
    rewards = torch.randn(b, generator=g, device="cuda", dtype=torch.float64)
    ranks = torch.randint(0, 4, (b,), generator=g, device="cuda")
    return obs, actions, masks, steps_to_done, rewards, ranks


GAMMA, MIN_Q, NEXT_RANK = 0.99, 5.0, 0.2


def torch_loss(brain, dqn, aux, bt, dtype=None):
    """mortal/train.py:228-247 (dtype float64 runs the models and the expressions in float64)"""
    obs, actions, masks, steps_to_done, rewards, ranks = bt
    q_target = (GAMMA ** steps_to_done * rewards).to(torch.float32)
    if dtype is not None:
        obs, q_target = obs.to(dtype), q_target.to(dtype)
    phi = brain(obs)
    q_out = dqn(phi, masks)
    q = q_out[range(obs.shape[0]), actions]
    dqn_loss = 0.5 * F.mse_loss(q, q_target)
    cql_loss = q_out.logsumexp(-1).mean() - q.mean()
    nr_loss = F.cross_entropy(aux(phi)[0], ranks)
    return dqn_loss + cql_loss * MIN_Q + nr_loss * NEXT_RANK


def fused_loss(brain, dqn, aux, bt):
    from mortal_b200 import train_ops

    obs, actions, masks, steps_to_done, rewards, ranks = bt
    phi = brain.forward_train(obs)
    v, a = dqn.heads(phi)
    dqn_loss, cql_loss, nr_loss, *_ = train_ops.dqn_losses(v, a, aux(phi)[0], masks, actions, steps_to_done, rewards, ranks, GAMMA)
    return dqn_loss + cql_loss * MIN_Q + nr_loss * NEXT_RANK


def grads(mods, loss, scale=1.0):
    params = [p for m in mods for p in m.parameters()]
    return [g.double() / scale for g in torch.autograd.grad(loss * scale, params)]


@pytest.fixture
def no_tf32():
    conv, mm = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = conv, mm


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("version,c,n,b", [(4, 192, 40, 32), (2, 32, 2, 16), (3, 32, 2, 16)])
def test_first_step_gradients_against_float64(version, c, n, b, dtype, no_tf32):
    base = models(version, c, n, seed=version)
    bt = batch(version, b, seed=version + 10, jitter=True)
    ref64 = [copy.deepcopy(m).double().train() for m in base]
    g64 = grads(ref64, torch_loss(*ref64, bt, torch.float64))
    amp = dtype == torch.float16
    scale = 1024.0 if amp else 1.0  # as GradScaler would: fp16 gradients of a deep net underflow unscaled
    tor, fus = [copy.deepcopy(m).train() for m in base], [copy.deepcopy(m).train() for m in base]
    with torch.autocast("cuda", enabled=amp):
        lt = torch_loss(*tor, bt)
    gt = grads(tor, lt, scale)
    with torch.autocast("cuda", enabled=amp):
        lf = fused_loss(*fus, bt)
    gf = grads(fus, lf, scale)
    names = [n_ for m in base for n_, _ in m.named_parameters()]
    eps = torch.finfo(dtype).eps
    for name, a, t, r in zip(names, gf, gt, g64):
        den = r.abs().max().item()
        e, et = ((a - r).abs().max().item() / den, (t - r).abs().max().item() / den) if den > 0 else (0.0, 0.0)
        assert e <= 2 * et + 8 * eps, f"{name}: fused e {e:.3e} > 2 * torch e {et:.3e} + 8 eps"
    # the running statistics the two forwards left behind
    for mt, mf, m64 in zip(tor[0].modules(), fus[0].modules(), ref64[0].modules()):
        if isinstance(mt, torch.nn.BatchNorm1d):
            assert int(mf.num_batches_tracked) == int(mt.num_batches_tracked) == 1
            for k in ("running_mean", "running_var"):
                r, t, f = getattr(m64, k), getattr(mt, k).double(), getattr(mf, k).double()
                den = r.abs().max().item()
                assert (f - r).abs().max().item() / den <= 2 * (t - r).abs().max().item() / den + 8 * eps, k


def test_adamw_steps_agree_with_torch_path():
    base = models(4, 64, 6, seed=7)
    arms = []
    for loss_fn in (torch_loss, fused_loss):
        ms = [copy.deepcopy(m).train() for m in base]
        opt = torch.optim.AdamW([p for m in ms for p in m.parameters()], lr=1e-4)
        losses = []
        for step in range(20):
            opt.zero_grad(set_to_none=True)
            loss = loss_fn(*ms, batch(4, 128, seed=100 + step % 5))
            loss.backward()
            opt.step()
            losses.append(loss.item())
        arms.append((ms, losses))
    (mt, lt), (mf, lf) = arms
    for step, (a, b) in enumerate(zip(lf, lt)):
        assert abs(a - b) <= 1e-3 * abs(b), f"step {step}: fused loss {a} vs torch {b}"
    for bt_, bf in zip(mt[0].modules(), mf[0].modules()):
        if isinstance(bt_, torch.nn.BatchNorm1d):
            assert int(bt_.num_batches_tracked) == int(bf.num_batches_tracked) == 20
            torch.testing.assert_close(bf.running_mean, bt_.running_mean, rtol=1e-3, atol=1e-4)
            torch.testing.assert_close(bf.running_var, bt_.running_var, rtol=1e-3, atol=1e-4)


def test_frozen_bn_leaves_running_statistics():
    brain, dqn, aux = models(4, 32, 2, seed=3)
    brain.freeze_bn(True)
    brain.train()
    before = {k: v.clone() for k, v in brain.state_dict().items() if "running" in k or "num_batches" in k}
    for step in range(3):
        fused_loss(brain, dqn, aux, batch(4, 64, seed=step)).backward()
    assert all(torch.equal(brain.state_dict()[k], v) for k, v in before.items())
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in brain.parameters())


# ---- train() -----------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def arena_logs(tmp_path_factory):
    from mortal_b200.libriichi.arena import OneVsThree

    d = tmp_path_factory.mktemp("arena_train")
    torch.manual_seed(5)
    OneVsThree(disable_progress_bar=True, log_dir=str(d / "logs")).py_vs_py(_Eng("alpha", 2.0), _Eng("beta", 0.5), (97000, 13), 4)
    return d


def tiny_cfg(root, name, logs):
    from mortal_b200.model import GRP, DQN, Brain, mortal_state_dict

    d = root / name
    d.mkdir(exist_ok=True)
    torch.manual_seed(11)
    torch.save({"model": GRP().state_dict()}, d / "grp.pth")
    b = Brain(conv_channels=32, num_blocks=2, version=4)
    torch.save({"mortal": mortal_state_dict(b), "current_dqn": DQN(version=4).state_dict(),
                "config": {"control": {"version": 4}, "resnet": {"conv_channels": 32, "num_blocks": 2}}}, d / "baseline.pth")
    return {
        "control": {"version": 4, "online": False, "batch_size": 128, "opt_step_every": 1, "save_every": 2, "test_every": 4,
                    "submit_every": 100, "device": "cuda:0", "enable_cudnn_benchmark": False, "enable_amp": False,
                    "enable_compile": False, "state_file": str(d / "mortal.pth"), "best_state_file": str(d / "best.pth"),
                    "tensorboard_dir": str(d / "tb")},
        "dataset": {"globs": [str(logs / "**" / "*.json.gz")], "file_index": str(d / "index.pth"), "file_batch_size": 4,
                    "reserve_ratio": 0.0, "num_workers": 1, "player_names_files": [], "num_epochs": 1,
                    "enable_augmentation": False, "augmented_first": False},
        "env": {"gamma": 1.0, "pts": [6.0, 4.0, 2.0, 0.0]},
        "resnet": {"conv_channels": 32, "num_blocks": 2},
        "cql": {"min_q_weight": 5.0},
        "aux": {"next_rank_weight": 0.2},
        "freeze_bn": {"mortal": False},
        "optim": {"eps": 1e-8, "betas": [0.9, 0.999], "weight_decay": 0.1, "max_grad_norm": 1.0,
                  "scheduler": {"peak": 1e-4, "final": 1e-5, "warm_up_steps": 2, "max_steps": 100}},
        "test_play": {"games": 8, "log_dir": str(d / "test_play")},
        "baseline": {"test": {"device": "cuda:0", "enable_compile": False, "state_file": str(d / "baseline.pth")}},
        "grp": {"network": {"hidden_size": 64, "num_layers": 2}, "state_file": str(d / "grp.pth")},
    }


STATE_KEYS = {"mortal", "current_dqn", "aux_net", "optimizer", "scheduler", "scaler", "steps", "timestamp", "best_perf", "config"}


@pytest.mark.parametrize("amp", [False, True])
def test_train_saves_tests_and_resumes(arena_logs, tmp_path, amp):
    from mortal_b200.engine import DeviceEngine
    from mortal_b200.libriichi.arena import OneVsThree
    from mortal_b200.model import load_mortal
    from mortal_b200.stat import Stat
    from mortal_b200.train import train

    cfg = tiny_cfg(tmp_path, "run", arena_logs / "logs")
    cfg["control"]["enable_amp"] = amp
    brain, dqn, aux, opt, steps = train(cfg, steps=4)
    assert steps == 4
    state = torch.load(cfg["control"]["state_file"], weights_only=True)
    assert set(state) == STATE_KEYS and state["steps"] == 4
    assert state["best_perf"]["avg_rank"] <= 4.0 and os.path.exists(cfg["control"]["best_state_file"])  # any result beats the start
    logs = os.listdir(cfg["test_play"]["log_dir"])
    assert len(logs) == 8
    assert isinstance(Stat.from_dir(cfg["test_play"]["log_dir"], "mortal", disable_progress_bar=True), Stat)
    b2, d2 = load_mortal(state)  # strict
    assert all(torch.equal(p.cpu(), q) for p, q in zip(brain.parameters(), b2.parameters()))
    eng = DeviceEngine(b2, d2, version=4, device=torch.device("cuda", 0), name="trained")
    OneVsThree(disable_progress_bar=True, log_dir=str(tmp_path / "play")).py_vs_py(eng, _Eng("beta", 0.5), (98000, 3), 1)
    assert len(os.listdir(tmp_path / "play")) == 4
    # resume: steps, optimizer, scheduler, scaler and best_perf come from the file
    _, _, _, opt2, steps2 = train(cfg, steps=2)
    assert steps2 == 6
    state2 = torch.load(cfg["control"]["state_file"], weights_only=True)
    assert state2["steps"] == 6 and state2["scheduler"]["last_epoch"] == 6
    assert all(s["step"].item() == 6 for s in state2["optimizer"]["state"].values())
    assert state2["best_perf"] == state["best_perf"]
    assert state2["scaler"].keys() == state["scaler"].keys() and ("scale" in state2["scaler"]) == amp  # {} when disabled


def test_illegal_action_raises(arena_logs, tmp_path, monkeypatch):
    from mortal_b200 import train as T

    class Corrupt(T.FileDatasetsIter):
        def __iter__(self):
            for i, (obs, actions, masks, *rest) in enumerate(super().__iter__()):
                if i == 0:
                    masks = masks.clone()
                    masks[0, actions[0]] = False
                yield (obs, actions, masks, *rest)

    monkeypatch.setattr(T, "FileDatasetsIter", Corrupt)
    cfg = tiny_cfg(tmp_path, "bad", arena_logs / "logs")
    with pytest.raises(ValueError, match="step 1"):
        T.train(cfg, steps=2)
    assert not os.path.exists(cfg["control"]["state_file"])


def _toml(d, prefix=""):
    out, tables = [], []
    for k, v in d.items():
        if isinstance(v, dict):
            tables.append((k, v))
        else:
            out.append(f"{k} = {_toml_value(v)}")
    for k, v in tables:
        name = f"{prefix}{k}"
        out.append(f"[{name}]")
        out.append(_toml(v, name + "."))
    return "\n".join(out)


def _toml_value(v):
    if isinstance(v, bool):
        return "true" if v else "false"
    if isinstance(v, str):
        return '"' + v.replace("\\", "\\\\") + '"'
    if isinstance(v, list):
        return "[" + ", ".join(_toml_value(x) for x in v) + "]"
    return repr(v)


def test_command_line(arena_logs, tmp_path):
    cfg = tiny_cfg(tmp_path, "cli", arena_logs / "logs")
    cfg["dataset"]["globs"] = [str(arena_logs / "logs" / sorted(os.listdir(arena_logs / "logs"))[0])]
    cfg["control"]["test_every"] = 1000
    (tmp_path / "tiny.toml").write_text(_toml(cfg))
    env = {**os.environ, "PYTHONPATH": ROOT}
    r = subprocess.run([sys.executable, "-m", "mortal_b200.train", str(tmp_path / "tiny.toml")], cwd=tmp_path, env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    state = torch.load(cfg["control"]["state_file"], weights_only=True)
    assert set(state) == STATE_KEYS and state["steps"] >= 2 and state["steps"] % 2 == 0
