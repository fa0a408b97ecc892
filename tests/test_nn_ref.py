"""The float64 references and bounds of nn_ref.py, checked on the CPU: composed, the per-op references are the stock network;
the bf16 spacing agrees with torch.nextafter; each bound accepts a correctly rounded result and rejects the next bf16 value out."""
import pytest
import torch

import nn_ref as R

BF16_MAX = float(torch.finfo(torch.bfloat16).max)


def _all_positive_bf16():
    bits = torch.arange(1, 0x7F80, dtype=torch.int32).to(torch.int16)  # every positive finite bf16 value, subnormals included
    return bits.view(torch.bfloat16)


def test_ulp_agrees_with_nextafter():
    x = _all_positive_bf16()
    up = torch.nextafter(x, torch.full_like(x, float("inf")))
    fin = torch.isfinite(up)
    assert torch.equal(R.ulp_bf16(x)[fin], (up.double() - x.double())[fin])
    down = torch.nextafter(x, torch.zeros_like(x))  # below a power of two the spacing halves: the ulp of the value below
    assert torch.equal(R.ulp_bf16(down.double()), x.double() - down.double())
    # subnormals, the smallest normal and powers of two, by value
    for v, u in ((2.0 ** -133, 2.0 ** -133), (2.0 ** -127, 2.0 ** -133), (2.0 ** -126, 2.0 ** -133), (2.0 ** -125, 2.0 ** -132),
                 (1.0, 2.0 ** -7), (1.0 - 2.0 ** -9, 2.0 ** -8), (3.0, 2.0 ** -6), (2.0 ** 127, 2.0 ** 120), (0.0, 2.0 ** -133)):
        assert R.ulp_bf16(torch.tensor([v, -v], dtype=torch.float64)).tolist() == [u, u], v
    assert torch.equal(R.half_ulp_bf16(x), R.ulp_bf16(x) / 2)


def _rounding_cases(n=20000, seed=0, lo=-30, hi=30):
    """float64 values spread over many binades, their correctly rounded bf16 value and the bf16 value one step further out"""
    g = torch.Generator().manual_seed(seed)
    v = torch.ldexp(1 + torch.rand(n, generator=g, dtype=torch.float64), torch.randint(lo, hi, (n,), generator=g, dtype=torch.int32))
    v = torch.where(torch.rand(n, generator=g) < 0.5, -v, v)
    v = torch.cat([v, torch.tensor([1e-40, -3e-39, 2.0 ** -126 * 1.3], dtype=torch.float64)])  # subnormal and near-subnormal
    r = R.rn_bf16(v)
    away = torch.where(r.double() > v, torch.full_like(r, float("inf")), torch.full_like(r, -float("inf")))
    away = torch.where(r.double() == v, torch.where(v > 0, away.abs(), -away.abs()), away)
    return v, r, torch.nextafter(r, away)


def _accepts_and_rejects(bound, v, r, out, slack, clear_share=0.9):
    """r is accepted everywhere; the next value out is rejected wherever v is not within `slack` (the bound's extra terms) of a
    bf16 value, where moving one value out does not have to leave the bound."""
    assert ((r.double() - v).abs() <= bound).all()
    clear = ((r.double() - v).abs() > 2 * slack)
    assert clear.float().mean() > clear_share
    assert ((out.double() - v).abs() > bound)[clear].all()


def test_bound_affine_mish_accepts_rn_and_rejects_one_out():
    v, r, out = _rounding_cases()
    b = R.bound_affine_mish(v)
    _accepts_and_rejects(b, v, r, out, 2.0 ** -16 * v.abs() + 2.0 ** -110)
    assert R.worst_violation(r, v, b)[0] <= 0 and R.worst_violation(out, v, b)[0] > 0


def test_bound_pool_mean_accepts_rn_and_rejects_one_out():
    v, r, out = _rounding_cases(seed=1)
    mean_abs = v.abs() * 3
    b = R.bound_pool_mean(v, mean_abs, 34)
    _accepts_and_rejects(b, v, r, out, 35 * 2.0 ** -24 * mean_abs)
    assert R.bound_pool_max(v).eq(0).all()


def test_bound_gate_accepts_rn_and_rejects_one_out():
    g = torch.Generator().manual_seed(2)
    v = torch.sigmoid(torch.randn(20000, generator=g, dtype=torch.float64) * 6)
    r = R.rn_bf16(v)
    away = torch.where(r.double() > v, torch.ones_like(r) * 2, torch.zeros_like(r) - 1)
    out = torch.nextafter(r, away)
    zabs = torch.rand(20000, generator=g, dtype=torch.float64) * 8
    b = R.bound_gate(v, zabs, 34, 192, 12)
    _accepts_and_rejects(b, v, r, out, b - R.half_ulp_bf16(v), clear_share=0.75)


def test_bound_conv_accepts_rn_and_rejects_one_out():
    v, r, out = _rounding_cases(seed=3)
    sum_abs = v.abs() * 2
    b = R.bound_conv(v, sum_abs, 192)
    _accepts_and_rejects(b, v, r, out, 576 * 2.0 ** -22 * sum_abs, clear_share=0.75)


def test_checkers_name_the_worst_element():
    v = torch.zeros(2, 8, 1, 3, dtype=torch.float64)
    got = R.rn_bf16(v)
    got[1, 5, 0, 2] = 1.0
    with pytest.raises(AssertionError, match=r"b=1, c=5, l=2"):
        R.check_within("t", got, v, R.bound_affine_mish(v), R.NHWC_DIMS)
    with pytest.raises(AssertionError, match=r"b=1, c=5, l=2"):
        R.check_bits("t", got, R.rn_bf16(v), R.NHWC_DIMS)
    # non-finite values: equal to the correctly rounded v, NaN by NaN-ness
    v = torch.tensor([float("nan"), float("inf"), -float("inf"), 1e39, -1e39, 2.0], dtype=torch.float64)
    got = torch.tensor([float("nan"), float("inf"), -float("inf"), float("inf"), -float("inf"), 2.0], dtype=torch.bfloat16)
    R.check_within("t", got, v, R.bound_affine_mish(v))
    for i, bad in ((0, 1.0), (1, BF16_MAX), (3, BF16_MAX), (5, float("nan"))):
        g2 = got.clone()
        g2[i] = bad
        assert R.worst_violation(g2, v, R.bound_affine_mish(v))[0] == float("inf"), i
    z = torch.tensor([0.0], dtype=torch.bfloat16)
    with pytest.raises(AssertionError):
        R.check_bits("t", z, -z)  # -0.0 differs from +0.0 by sign


def _randomise_bn(brain, seed):
    g = torch.Generator().manual_seed(seed)
    for m in brain.modules():
        if isinstance(m, torch.nn.BatchNorm1d):
            m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.1)
            m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) + 0.5)
            m.weight.data.copy_(torch.rand(m.weight.shape, generator=g) + 0.5)
            m.bias.data.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)


def compose_brain(brain, obs):
    """Brain.forward restated with the per-op references (BN folded to its affine, float64 throughout)"""
    from mortal_b200.model import PreActBlock

    aff = lambda bn: tuple(t.flatten() for t in PreActBlock._affine(bn))
    x, _ = R.conv1x3(R.stem_input(obs, obs.shape[1]), brain.stem.weight)
    for blk in brain.blocks:
        y, _ = R.conv1x3(R.affine_mish(x, *aff(blk.bn1)), blk.conv1.weight)
        y, _ = R.conv1x3(R.affine_mish(y, *aff(blk.bn2)), blk.conv2.weight)
        g, _ = R.gate(y, blk.gate.fc1.weight, blk.gate.fc1.bias, blk.gate.fc2.weight.T, blk.gate.fc2.bias)
        x = R.gate_residual(y, g, x)
    x, _ = R.conv1x3(R.affine_mish(x, *aff(brain.bn)), brain.neck.weight, brain.neck.bias)
    x = R.mish(x).flatten(1)
    return R.mish(x @ R.f64(brain.fc.weight).T + R.f64(brain.fc.bias))


def test_composed_references_equal_brain_forward():
    from mortal_b200.model import Brain

    torch.manual_seed(0)
    brain = Brain(conv_channels=32, num_blocks=3).double().eval()
    _randomise_bn(brain, 1)
    for blk in brain.blocks:  # non-zero gate biases, so that b1 / b2 are exercised
        blk.gate.fc1.bias.data.normal_(0, 0.3)
        blk.gate.fc2.bias.data.normal_(0, 0.3)
    obs = (torch.rand(5, 1012, 34, dtype=torch.float64) < 0.1).double()
    with torch.no_grad():
        ref = brain(obs)
        got = compose_brain(brain, obs)
    assert ref.shape == got.shape == (5, 1024)
    assert ((got - ref).abs() <= 1e-12 * ref.abs().max()).all(), (got - ref).abs().max().item()


def test_pool_and_gate_references_by_hand():
    y = torch.tensor([[1.0, -2.0, 4.0], [-1.0, -3.0, -0.5]], dtype=torch.float64).view(1, 2, 1, 3)
    mean, mx = R.pool_mean_max(y)
    assert mean.tolist() == [[1.0, -1.5]] and mx.tolist() == [[4.0, -0.5]]
    w1 = torch.tensor([[1.0, -1.0]], dtype=torch.float64)
    b1 = torch.tensor([0.5], dtype=torch.float64)
    w2t = torch.tensor([[2.0, -0.5]], dtype=torch.float64)
    b2 = torch.tensor([0.1, -0.1], dtype=torch.float64)
    g, zabs = R.gate(y, w1, b1, w2t, b2)
    m = lambda p: p * torch.tanh(torch.nn.functional.softplus(torch.tensor(p, dtype=torch.float64)))
    ha, hm = m(1.0 + 1.5 + 0.5), m(4.0 + 0.5 + 0.5)
    z = torch.stack([2 * ha + 0.1 + 2 * hm + 0.1, -0.5 * ha - 0.1 - 0.5 * hm - 0.1])
    assert torch.allclose(g[0], torch.sigmoid(z), rtol=1e-15, atol=0)
    pa, pm = 1 + 1.5 + 0.5, 4 + 0.5 + 0.5
    assert torch.allclose(zabs[0], torch.tensor([2 * pa + 0.1 + 2 * pm + 0.1, 0.5 * pa + 0.1 + 0.5 * pm + 0.1], dtype=torch.float64))
