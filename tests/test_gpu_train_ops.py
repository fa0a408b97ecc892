"""The policy net's fused training kernels (csrc/mjx_train.cuh, mortal_b200.train_ops) against float64 torch autograd of the same
operation on the kernels' own inputs. With e = |got - ref64|_inf / |ref64|_inf, every output and gradient of the fused path must
have e <= 2 * (torch's own e at the same storage dtype) + 8 * finfo(dtype).eps. Shapes B in {1, 3, 512, 4096}, C in {8, 32, 192,
256}, float32 and float16 (autocast), train and frozen BatchNorm, with a constant channel, a channel of mean 1e3 and std 0.1, tied
maxima, rows with one and with all 46 legal actions, gamma 1 and 0.99 with steps_to_done up to 300; non-finite upstream gradients
reach the parameter gradients (GradScaler skips the step); repeats are bit-identical."""
from __future__ import annotations

import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import torch.nn.functional as F  # noqa: E402

BS = (1, 3, 512, 4096)
CS = (8, 32, 192, 256)
DTYPES = (torch.float32, torch.float16)
L = 34


def err(got, ref):
    got, ref = got.double(), ref.double()
    den = ref.abs().max().item()
    d = (got - ref).abs().max().item()
    return d / den if den > 0 else d


def check(name, got, ref64, torch_got, dtype):
    e, et = err(got, ref64), err(torch_got, ref64)
    bound = 2 * et + 8 * torch.finfo(dtype).eps
    assert e <= bound, f"{name}: fused e {e:.3e} > 2 * torch e {et:.3e} + 8 eps ({bound:.3e})"


def activations(b, c, dtype, seed, quantize=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((b, c, 1, L), generator=g, device="cuda") * 1.5 + 0.3
    x[:, 0] = 0.75  # a constant channel: variance 0
    if c > 1:
        x[:, 1] = 1e3 + 0.1 * torch.randn((b, 1, L), generator=g, device="cuda")  # a one-pass variance fails here
    if quantize:
        x = (x * 4).round() / 4  # many tied maxima in each pooling window
    return x.to(dtype).contiguous(memory_format=torch.channels_last)


def make_bn(c, seed):
    torch.manual_seed(seed)
    bn = torch.nn.BatchNorm1d(c, momentum=0.01, eps=1e-3).cuda()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.normal_(0, 0.3)
        bn.running_mean.normal_(0, 0.2)
        bn.running_var.uniform_(0.5, 1.5)
    return bn


def bn_mish_ref(x, bn, training, dout, dtype64=torch.float64, amp=False):
    """torch's BatchNorm1d + Mish on [B, C, L] in dtype64 (float64: the reference) or at the storage dtype; returns (out, dx,
    dgamma, dbeta, running_mean, running_var)"""
    w = bn.weight.detach().to(dtype64 if dtype64 == torch.float64 else torch.float32).requires_grad_()
    b = bn.bias.detach().to(w.dtype).requires_grad_()
    rm, rv = bn.running_mean.clone().to(w.dtype), bn.running_var.clone().to(w.dtype)
    xi = x.detach().squeeze(2).to(dtype64 if dtype64 == torch.float64 else x.dtype).requires_grad_()
    with torch.autocast("cuda", enabled=amp):
        out = F.mish(F.batch_norm(xi, rm, rv, w, b, training, bn.momentum, bn.eps))
    dx, dw, db = torch.autograd.grad(out, (xi, w, b), dout.squeeze(2).to(out.dtype))
    return out.unsqueeze(2), dx.unsqueeze(2), dw, db, rm, rv


@pytest.mark.parametrize("frozen", [False, True])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("c", CS)
@pytest.mark.parametrize("b", BS)
def test_bn_mish_against_float64(b, c, dtype, frozen):
    from mortal_b200 import train_ops

    x = activations(b, c, dtype, seed=b * 1000 + c)
    bn = make_bn(c, seed=c)
    dout = activations(b, c, dtype, seed=b * 1000 + c + 7) * 0.1
    dout[:, 1] = 0.05  # not 1e3
    ref = bn_mish_ref(x, bn, not frozen, dout)
    tor = bn_mish_ref(x, bn, not frozen, dout, dtype64=dtype, amp=dtype == torch.float16)
    xi = x.detach().requires_grad_()
    bn.train()
    n0 = int(bn.num_batches_tracked)
    out = train_ops.bn_mish(xi, bn, frozen=frozen)
    dx, dw, db = torch.autograd.grad(out, (xi, bn.weight, bn.bias), dout)
    assert out.dtype == dtype and dx.dtype == dtype and dw.dtype == torch.float32
    for name, i, got in (("out", 0, out), ("dx", 1, dx), ("dgamma", 2, dw), ("dbeta", 3, db), ("running_mean", 4, bn.running_mean),
                         ("running_var", 5, bn.running_var)):
        check(name, got, ref[i], tor[i], dtype)
    assert int(bn.num_batches_tracked) == n0 + (0 if frozen else 1)
    if frozen:
        assert torch.equal(bn.running_mean, ref[4].float()) and torch.equal(bn.running_var, ref[5].float())


class _Gate(torch.nn.Module):
    def __init__(self, c):
        super().__init__()
        from mortal_b200.model import ChannelGate

        self.gate = ChannelGate(c)
        with torch.no_grad():
            for p in self.gate.parameters():
                p.normal_(0, 0.3)


def gate_ref(y, x, gate, dout, dtype64, amp):
    """ChannelGate(y) + x in torch (mortal/model.py ChannelAttention + residual) on [B, C, L]: (out, dy, dx, dW1, db1, dW2, db2)"""
    params = [p.detach().to(dtype64 if dtype64 == torch.float64 else torch.float32).requires_grad_() for p in
              (gate.fc1.weight, gate.fc1.bias, gate.fc2.weight, gate.fc2.bias)]
    yi = y.detach().squeeze(2).to(dtype64 if dtype64 == torch.float64 else y.dtype).requires_grad_()
    xi = x.detach().squeeze(2).to(yi.dtype).requires_grad_()
    w1, b1, w2, b2 = params
    mlp = lambda v: F.linear(F.mish(F.linear(v, w1, b1)), w2, b2)
    with torch.autocast("cuda", enabled=amp):
        g = torch.sigmoid(mlp(yi.mean(-1)) + mlp(yi.amax(-1)))
        out = yi * g.unsqueeze(-1) + xi
    grads = torch.autograd.grad(out, (yi, xi, *params), dout.squeeze(2).to(out.dtype))
    return (out.unsqueeze(2), grads[0].unsqueeze(2), grads[1].unsqueeze(2), *grads[2:])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("c", CS)
@pytest.mark.parametrize("b", BS)
def test_gate_residual_against_float64(b, c, dtype):
    from mortal_b200 import train_ops

    gate = _Gate(c).cuda().gate
    y = activations(b, c, dtype, seed=b + c, quantize=True)
    y[:, 1] = (y[:, 1].float() - 1e3).to(dtype)
    x = activations(b, c, dtype, seed=b + c + 1)
    dout = activations(b, c, dtype, seed=b + c + 2) * 0.1
    dout[:, 1] = 0.05
    ref = gate_ref(y, x, gate, dout, torch.float64, False)
    tor = gate_ref(y, x, gate, dout, dtype, dtype == torch.float16)
    yi, xi = y.detach().requires_grad_(), x.detach().requires_grad_()
    params = [gate.fc1.weight, gate.fc1.bias, gate.fc2.weight, gate.fc2.bias]
    with torch.autocast("cuda", enabled=dtype == torch.float16):
        out = train_ops.gate_residual(yi, xi, gate)
    grads = torch.autograd.grad(out, (yi, xi, *params), dout, allow_unused=True)
    got = (out, *grads)
    for name, i in (("out", 0), ("dy", 1), ("dx", 2), ("dW1", 3), ("db1", 4), ("dW2", 5), ("db2", 6)):
        if ref[i].numel() == 0:
            continue  # C = 8: the gate's hidden layer has 8 // 16 = 0 units
        check(name, got[i], ref[i], tor[i], dtype)


def loss_inputs(b, dtype, gamma_seed):
    g = torch.Generator(device="cuda").manual_seed(gamma_seed)
    v = torch.randn((b, 1), generator=g, device="cuda").to(dtype)
    a = torch.randn((b, 46), generator=g, device="cuda").to(dtype)
    aux = torch.randn((b, 4), generator=g, device="cuda").to(dtype)
    masks = torch.rand((b, 46), generator=g, device="cuda") < 0.3
    masks[torch.arange(b, device="cuda"), torch.randint(0, 46, (b,), generator=g, device="cuda")] = True
    masks[0] = False
    masks[0, 17] = True  # one legal action
    if b > 1:
        masks[1] = True  # all 46 legal
    actions = torch.multinomial(masks.float(), 1, generator=g).squeeze(1)
    steps_to_done = torch.randint(0, 301, (b,), generator=g, device="cuda")
    steps_to_done[0] = 300
    rewards = torch.randn(b, generator=g, device="cuda", dtype=torch.float64) * 3
    ranks = torch.randint(0, 4, (b,), generator=g, device="cuda")
    return v, a, aux, masks, actions, steps_to_done, rewards, ranks


def loss_ref(v, a, aux, masks, actions, steps_to_done, rewards, ranks, gamma, wts, dtype64, amp):
    """mortal/train.py:228-247 in torch with DQN.forward's masked combine: (dqn, cql, next_rank, q, q_target, dv, da, daux)"""
    dt = dtype64 if dtype64 == torch.float64 else v.dtype
    vi, ai, xi = (t.detach().to(dt).requires_grad_() for t in (v, a, aux))
    q_target = (gamma ** steps_to_done * rewards).to(torch.float32)
    b = v.shape[0]
    with torch.autocast("cuda", enabled=amp):
        a_mean = ai.masked_fill(~masks, 0.0).sum(-1, keepdim=True) / masks.sum(-1, keepdim=True)
        q_out = (vi + ai - a_mean).masked_fill(~masks, -torch.inf)
        q = q_out[torch.arange(b), actions]
        dqn = 0.5 * F.mse_loss(q, q_target.to(q.dtype) if dt == torch.float64 else q_target)
        cql = q_out.logsumexp(-1).mean() - q.mean()
        nr = F.cross_entropy(xi, ranks)
        loss = dqn * wts[0] + cql * wts[1] + nr * wts[2]
    dv, da, dx = torch.autograd.grad(loss, (vi, ai, xi))
    return dqn, cql, nr, q, q_target, dv, da, dx


@pytest.mark.parametrize("gamma", [1.0, 0.99])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b", BS)
def test_dqn_losses_against_float64(b, dtype, gamma):
    from mortal_b200 import train_ops

    inputs = loss_inputs(b, dtype, gamma_seed=b)
    wts = (1.0, 0.4, 0.2)
    ref = loss_ref(*inputs, gamma, wts, torch.float64, False)
    tor = loss_ref(*inputs, gamma, wts, dtype, dtype == torch.float16)
    v, a, aux = (t.detach().requires_grad_() for t in inputs[:3])
    dqn, cql, nr, q, q_target, bad = train_ops.dqn_losses(v, a, aux, *inputs[3:], gamma)
    assert int(bad) == 0
    assert torch.equal(q_target, tor[4]), "q_target is torch's float32 expression, bit for bit"
    loss = dqn * wts[0] + cql * wts[1] + nr * wts[2]
    dv, da, daux = torch.autograd.grad(loss, (v, a, aux))
    for name, i, got in (("dqn_loss", 0, dqn), ("cql_loss", 1, cql), ("next_rank_loss", 2, nr), ("q", 3, q), ("dv", 5, dv),
                         ("da", 6, da), ("daux", 7, daux)):
        check(name, got, ref[i], tor[i], dtype)


def test_dqn_losses_flags_an_illegal_action():
    from mortal_b200 import train_ops

    inputs = list(loss_inputs(64, torch.float32, gamma_seed=5))
    masks, actions = inputs[3].clone(), inputs[4]
    masks[10, actions[10]] = False
    masks[10, (actions[10] + 1) % 46] = True
    inputs[3] = masks
    *_, bad = train_ops.dqn_losses(*inputs, 0.99)
    assert int(bad) != 0


def test_repeats_are_bit_identical():
    from mortal_b200 import train_ops

    b, c = 512, 192
    bn1, bn2 = make_bn(c, 1), make_bn(c, 1)
    gate = _Gate(c).cuda().gate
    x = activations(b, c, torch.float32, seed=11)
    dout = activations(b, c, torch.float32, seed=12) * 0.1
    runs = []
    for bn in (bn1, bn2):
        xi = x.detach().requires_grad_()
        out = train_ops.gate_residual(train_ops.bn_mish(xi, bn), xi, gate)
        grads = torch.autograd.grad(out, (xi, bn.weight, bn.bias, gate.fc1.weight, gate.fc2.weight), dout)
        runs.append((out, *grads, bn.running_mean.clone(), bn.running_var.clone()))
    inputs = loss_inputs(512, torch.float32, gamma_seed=3)
    for _ in range(2):
        v, a, aux = (t.detach().requires_grad_() for t in inputs[:3])
        dqn, cql, nr, q, qt, _ = train_ops.dqn_losses(v, a, aux, *inputs[3:], 0.99)
        runs.append((dqn, cql, nr, q, qt, *torch.autograd.grad(dqn + cql + nr, (v, a, aux))))
    for r0, r1 in ((runs[0], runs[1]), (runs[2], runs[3])):
        assert all(torch.equal(p, q) for p, q in zip(r0, r1))


def test_non_finite_gradient_reaches_parameters_and_scaler_skips():
    from mortal_b200 import train_ops

    b, c = 64, 32
    bn = make_bn(c, 2)
    gate = _Gate(c).cuda().gate
    x = activations(b, c, torch.float16, seed=21)
    params = [bn.weight, bn.bias, *gate.parameters()]
    before = [p.detach().clone() for p in params]
    opt = torch.optim.SGD(params, lr=0.1)
    scaler = torch.amp.GradScaler("cuda")
    scale0 = scaler.get_scale()
    with torch.autocast("cuda"):
        out = train_ops.gate_residual(train_ops.bn_mish(x, bn), x, gate)
        w = torch.ones_like(out)
        w[3, 5, 0, 7] = torch.inf
        loss = (out.float() * w.float()).sum()
    scaler.scale(loss).backward()
    assert not torch.isfinite(bn.weight.grad).all() and not torch.isfinite(bn.bias.grad).all()
    assert not torch.isfinite(gate.fc2.bias.grad).all()
    scaler.step(opt)
    scaler.update()
    assert all(torch.equal(p, q) for p, q in zip(params, before)), "GradScaler must skip the step"
    assert scaler.get_scale() < scale0


def test_rejections():
    from mortal_b200 import train_ops

    bn = make_bn(12, 0)
    with pytest.raises(ValueError):
        train_ops.bn_mish(torch.zeros((4, 12, 1, L), device="cuda"), bn)
    bn = make_bn(264, 0)
    with pytest.raises(ValueError):
        train_ops.bn_mish(torch.zeros((4, 264, 1, L), device="cuda"), bn)
    bn = make_bn(16, 0)
    with pytest.raises(ValueError):
        train_ops.bn_mish(torch.zeros((4, 16, 1, L), device="cuda", dtype=torch.bfloat16), bn)
    with pytest.raises(ValueError):
        train_ops.bn_mish(torch.zeros((0, 16, 1, L), device="cuda"), bn)
