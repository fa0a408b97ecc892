"""The policy-net trainer's host side (no GPU): mortal_state_dict against the reference's key layout pinned in
tests/golden/mortal_model_outputs.npz and its round trip through load_mortal, the optimizer's parameter groups in the reference's
sorted-name order, the learning-rate schedule and its state_dict keys, Brain.freeze_bn, AuxNet, and the config rejections."""
from __future__ import annotations

import math

import pytest

torch = pytest.importorskip("torch")

import mortal_ckpt as M  # noqa: E402


@pytest.fixture(scope="module")
def fixture():
    return M.load_fixture()


@pytest.mark.parametrize("name", ["v2", "v3", "v4"])
def test_mortal_state_dict_has_reference_keys_and_loads_back(fixture, name):
    from mortal_b200.model import load_mortal, mortal_state_dict

    fx = fixture[name]
    brain, dqn = load_mortal(M.checkpoint(name, fx))
    sd = mortal_state_dict(brain)
    assert [(k, list(v.shape)) for k, v in sd.items()] == [(k, list(s)) for k, s in fx["brain_keys"]]
    ref = M.checkpoint(name, fx)["mortal"]
    assert all(torch.equal(sd[k], ref[k]) for k in ref)
    b2, _ = load_mortal({"mortal": sd, "current_dqn": dqn.state_dict(), "config": M.config(brain.version)})
    assert all(torch.equal(p, q) for p, q in zip(brain.state_dict().values(), b2.state_dict().values()))


def test_mortal_state_dict_round_trip_192x40():
    from mortal_b200.model import DQN, Brain, load_mortal, load_mortal_state, mortal_state_dict

    torch.manual_seed(0)
    brain = Brain(conv_channels=192, num_blocks=40, version=4)
    with torch.no_grad():
        for m in brain.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.running_mean.normal_()
                m.running_var.uniform_(0.5, 2)
                m.num_batches_tracked.fill_(7)
    sd = mortal_state_dict(brain)
    assert next(iter(sd)) == "encoder.net.0.weight" and "encoder.net.40.res_unit.5.weight" in sd and "encoder.net.46.bias" in sd
    cfg = {"control": {"version": 4}, "resnet": {"conv_channels": 192, "num_blocks": 40}}
    b2, _ = load_mortal({"mortal": sd, "current_dqn": DQN(version=4).state_dict(), "config": cfg})
    b3 = Brain(conv_channels=192, num_blocks=40, version=4)
    load_mortal_state(b3, sd)
    assert all(torch.equal(p, q) for p, q in zip(brain.state_dict().values(), b3.state_dict().values()))  # resuming: all of it
    assert all(torch.equal(v, b2.state_dict()[k]) for k, v in brain.state_dict().items() if not k.endswith("num_batches_tracked"))
    with pytest.raises(KeyError):
        load_mortal_state(b3, {k: v for k, v in sd.items() if not k.startswith("encoder.net.46")})


def test_optimizer_groups_follow_sorted_reference_names():
    from mortal_b200.model import DQN, AuxNet, Brain, mortal_state_dict
    from mortal_b200.train import make_optimizer, named_param_groups

    for version in (2, 3, 4):
        brain, dqn, aux = Brain(conv_channels=32, num_blocks=3, version=version), DQN(version=version), AuxNet((4,))
        decay, no_decay = named_param_groups(brain, dqn, aux)
        brain_keys = mortal_state_dict(brain)
        want_decay, want_no = [], []
        for names, is_bn in (([k for k in brain_keys if "running" not in k and "num_batches" not in k],
                              lambda k: k.rsplit(".", 1)[0] + ".running_mean" in brain_keys),
                             (list(dqn.state_dict()), lambda k: False), (list(aux.state_dict()), lambda k: False)):
            # the reference: Linear / Conv1d weights decay; a BatchNorm's weight (running statistics beside it) does not
            dec = sorted(k for k in names if k.endswith("weight") and not is_bn(k))
            want_decay += dec
            want_no += sorted(set(names) - set(dec))
        assert [n for n, _ in decay] == want_decay
        assert [n for n, _ in no_decay] == want_no
        opt = make_optimizer(brain, dqn, aux, {"weight_decay": 0.1, "betas": [0.9, 0.999], "eps": 1e-8})
        assert opt.param_groups[0]["weight_decay"] == 0.1 and opt.param_groups[1]["weight_decay"] == 0
        assert opt.param_groups[0]["lr"] == 1
        assert [id(p) for p in opt.param_groups[0]["params"]] == [id(p) for _, p in decay]
        assert [id(p) for p in opt.param_groups[1]["params"]] == [id(p) for _, p in no_decay]


def _formula(step, init, peak, final, warm_up_steps, max_steps, offset=0, epoch_size=0):
    step += offset
    if epoch_size > 0:
        step %= epoch_size
    if warm_up_steps > 0 and step < warm_up_steps:
        return init + (peak - init) / warm_up_steps * step
    if step < max_steps:
        return final + 0.5 * (peak - final) * (1 + math.cos((step - warm_up_steps) / (max_steps - warm_up_steps) * math.pi))
    return final


@pytest.mark.parametrize("kw", [dict(peak=1e-3, final=1e-4, warm_up_steps=10, max_steps=50),
                                dict(peak=1e-3, final=1e-4, warm_up_steps=10, max_steps=50, init=1e-6, offset=3, epoch_size=37),
                                dict(peak=5e-4, final=5e-4, warm_up_steps=0, max_steps=20)])
def test_scheduler_matches_formula(kw):
    from mortal_b200.lr_scheduler import LinearWarmUpCosineAnnealingLR

    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.AdamW([p], lr=1)
    sched = LinearWarmUpCosineAnnealingLR(opt, **kw)
    full = {"init": 1e-8, **kw}
    for step in range(80):  # warm-up, cosine, past max_steps, and the epoch_size wrap
        assert sched.get_last_lr()[0] == _formula(step, **full), step
        opt.step()
        sched.step()
    sd = sched.state_dict()
    assert {"init", "peak", "final", "warm_up_steps", "max_steps", "offset", "epoch_size", "base_lrs", "last_epoch"} <= set(sd)
    assert sd["last_epoch"] == 80
    s2 = LinearWarmUpCosineAnnealingLR(torch.optim.AdamW([p], lr=1), **kw)
    s2.load_state_dict(sd)
    assert s2.last_epoch == 80 and s2.get_last_lr() == sched.get_last_lr()


def test_freeze_bn_and_aux_net():
    from mortal_b200.model import AuxNet, Brain

    brain = Brain(conv_channels=16, num_blocks=2, version=4)
    brain.freeze_bn(True)
    brain.train()
    assert brain.training and not any(m.training for m in brain.modules() if isinstance(m, torch.nn.BatchNorm1d))
    brain.freeze_bn(False)
    assert all(m.training for m in brain.modules())
    with torch.no_grad():
        brain.bn.running_mean.fill_(3)
    brain.reset_running_stats()
    assert torch.equal(brain.bn.running_mean, torch.zeros(16))
    aux = AuxNet((4,))
    assert list(aux.state_dict()) == ["net.weight"] and aux.net.bias is None
    out = aux(torch.zeros(2, 1024))
    assert isinstance(out, tuple) and out[0].shape == (2, 4)


def _cfg(**control):
    return {"control": {"version": 4, "online": False, "save_every": 2, "opt_step_every": 1, "test_every": 4, **control},
            "resnet": {"conv_channels": 192, "num_blocks": 40}}


def test_config_rejections():
    from mortal_b200.train import check_config, train

    check_config(_cfg())
    with pytest.raises(ValueError, match="online"):
        train(_cfg(online=True))
    with pytest.raises(ValueError, match="version 1"):
        train(_cfg(version=1))
    bad = _cfg()
    bad["resnet"]["conv_channels"] = 36
    with pytest.raises(ValueError, match="multiple of 8"):
        train(bad)
