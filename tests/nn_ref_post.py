"""float64 references and error bounds for the version-1 (post-activation) and oracle-stem kernels of csrc/mjx_nn.cuh, in the
style of nn_ref.py: each takes the kernel's actual inputs and computes the operation in float64."""
from __future__ import annotations

import torch

import nn_ref as R


def affine_relu(x, scale, bias):
    """relu(x * scale[c] + bias[c]), the pre-activation taken as the ±inf fp32 makes of it beyond the fp32 range; NaN stays NaN"""
    t = R.pre_activation(x, scale, bias)
    t32 = t.to(torch.float32)
    return torch.relu(torch.where(torch.isinf(t32) & torch.isfinite(t), R.f64(t32), t))


def bound_affine_relu(v):
    """one fp32 FMA (2^-24 relative) and the rounding to bf16 (half an ulp); relu is exact"""
    v = R.f64(v)
    return R.half_ulp_bf16(v) + 2.0 ** -24 * v.abs()


def post_gate(y, scale, bias, w1, b1, w2t, b2):
    """The post-activation block's gate: t = y * scale + bias, sigmoid(mlp(mean_L t) + mlp(max_L t)), mlp(v) = w2 relu(w1 v + b1)
    + b2. Returns (g, zabs): zabs is z with every term by its absolute value, pooled from |t| (mean |t|, max |t|)."""
    t = R.pre_activation(y, scale, bias).flatten(2)
    w1, b1, w2t, b2 = R.f64(w1), R.f64(b1), R.f64(w2t), R.f64(b2)
    z = zabs = 0
    for v, va in ((t.mean(-1), t.abs().mean(-1)), (t.amax(-1), t.abs().amax(-1))):
        z = z + torch.relu(v @ w1.T + b1) @ w2t + b2
        zabs = zabs + ((va @ w1.abs().T + b1.abs()) @ w2t.abs() + b2.abs())
    return torch.sigmoid(z), zabs


def bound_post_gate(g, zabs, length, channels, hidden):
    """nn_ref.bound_gate with two more fp32 roundings per pooled value (the affine's FMA)"""
    return R.bound_gate(g, zabs, length + 2, channels, hidden)


def post_residual(y, scale, bias, g, x):
    """relu((y * scale + bias) * g + x) for the kernel's bf16 gate g [B, C]; also the scale |t| g + |x| of its fp32 error"""
    t = R.pre_activation(y, scale, bias)
    gg = R.f64(g).view(g.shape[0], g.shape[1], 1, 1)
    return torch.relu(t * gg + R.f64(x)), t.abs() * gg + R.f64(x).abs()


def bound_post_residual(v, scale_abs):
    """the affine FMA and the gate FMA, 2^-24 of |t| g + |x| each, and half an ulp for bf16"""
    return R.half_ulp_bf16(v) + 2.0 ** -23 * R.f64(scale_abs)


def stem_input2(obs, obs2, channels_padded):
    """torch.cat((obs, obs2), 1) zero-padded to channels_padded, as float64 [B, channels_padded, 1, L]"""
    return R.stem_input(torch.cat((obs, obs2), 1), channels_padded)
