"""ctypes wrappers of the fused policy-net kernels in libmjx (csrc/mjx_nn.cuh). Tensors are CUDA bf16, logically
[B, C, 1, L] in channels_last memory format, i.e. [B, L, C] in memory. Every tensor handed to a kernel must start on a
16-byte boundary (the kernels read 16-byte vectors): a view at an odd offset into a larger buffer is refused here."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib


def _stream(t: torch.Tensor):
    return C.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def _aligned(*ts: torch.Tensor):
    for t in ts:
        assert t.is_cuda and t.data_ptr() % 16 == 0, "nn_ops: tensors must be CUDA and 16-byte aligned"


def _check_nhwc(x: torch.Tensor):
    assert x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 4 and x.shape[2] == 1
    b, c, _, l = x.shape
    assert c % 8 == 0 and x.stride(1) == 1 and x.stride(3) == c and x.stride(0) == c * l, "expected channels_last [B, C, 1, L]"
    _aligned(x)
    return b, c, l


def affine_mish(x: torch.Tensor, scale: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """mish(x * scale[c] + bias[c]); scale / bias float32 [C]"""
    b, c, l = _check_nhwc(x)
    assert scale.dtype == torch.float32 and bias.dtype == torch.float32 and scale.numel() == c == bias.numel()
    assert scale.is_contiguous() and bias.is_contiguous()
    _aligned(scale, bias)
    out = torch.empty_like(x)
    _lib.check(_lib.load().mjx_nn_affine_mish_bf16(C.c_void_p(x.data_ptr()), C.c_void_p(scale.data_ptr()), C.c_void_p(bias.data_ptr()),
                                                   C.c_void_p(out.data_ptr()), x.numel(), c, _stream(x)), "mjx_nn_affine_mish_bf16")
    return out


def affine_relu(x: torch.Tensor, scale: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """relu(x * scale[c] + bias[c]); scale / bias float32 [C] (version 1's BatchNorm + ReLU)"""
    b, c, l = _check_nhwc(x)
    assert scale.dtype == torch.float32 and bias.dtype == torch.float32 and scale.numel() == c == bias.numel()
    assert scale.is_contiguous() and bias.is_contiguous()
    _aligned(scale, bias)
    out = torch.empty_like(x)
    _lib.check(_lib.load().mjx_nn_affine_relu_bf16(C.c_void_p(x.data_ptr()), C.c_void_p(scale.data_ptr()), C.c_void_p(bias.data_ptr()),
                                                   C.c_void_p(out.data_ptr()), x.numel(), c, _stream(x)), "mjx_nn_affine_relu_bf16")
    return out


def pool_mean_max(x: torch.Tensor):
    """(mean over L, max over L) -> two bf16 [B, C] tensors"""
    b, c, l = _check_nhwc(x)
    avg = torch.empty((b, c), dtype=torch.bfloat16, device=x.device)
    mx = torch.empty((b, c), dtype=torch.bfloat16, device=x.device)
    _lib.check(_lib.load().mjx_nn_pool_bf16(C.c_void_p(x.data_ptr()), C.c_void_p(avg.data_ptr()), C.c_void_p(mx.data_ptr()), b, l, c,
                                            _stream(x)), "mjx_nn_pool_bf16")
    return avg, mx


def gate_residual(y: torch.Tensor, gate: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """y * gate[b, c] + x; gate bf16 [B, C] contiguous"""
    b, c, l = _check_nhwc(y)
    assert _check_nhwc(x) == (b, c, l) and gate.dtype == torch.bfloat16 and gate.shape == (b, c) and gate.is_contiguous()
    _aligned(gate)
    out = torch.empty_like(y)
    _lib.check(_lib.load().mjx_nn_gate_residual_bf16(C.c_void_p(y.data_ptr()), C.c_void_p(gate.data_ptr()), C.c_void_p(x.data_ptr()),
                                                     C.c_void_p(out.data_ptr()), b, l, c, _stream(y)), "mjx_nn_gate_residual_bf16")
    return out


def block_tail(y: torch.Tensor, x: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor, w2t: torch.Tensor, b2: torch.Tensor,
               scale: torch.Tensor, bias: torch.Tensor):
    """Channel gate + residual + the next pre-activation: gate = sigmoid(mlp(mean_L y) + mlp(max_L y)) with
    mlp(v) = w2 @ mish(w1 @ v + b1) + b2 (float32: w1 [H, C], w2t = w2.T [H, C]); returns (y * gate + x, mish((y * gate + x) * scale + bias))."""
    b, c, l = _check_nhwc(y)
    assert _check_nhwc(x) == (b, c, l)
    h = w1.shape[0]
    for t, shape in ((w1, (h, c)), (b1, (h,)), (w2t, (h, c)), (b2, (c,)), (scale, (c,)), (bias, (c,))):
        assert t.dtype == torch.float32 and tuple(t.shape) == shape and t.is_contiguous() and t.is_cuda
    _aligned(w1, b1, w2t, b2, scale, bias)
    assert c <= 256, "block_tail: at most 256 channels"
    x_out, a_out = torch.empty_like(y), torch.empty_like(y)
    gate = torch.empty((b, c), dtype=torch.bfloat16, device=y.device)
    p = lambda t: C.c_void_p(t.data_ptr())
    _lib.check(_lib.load().mjx_nn_block_tail_bf16(p(y), p(x), p(w1), p(b1), p(w2t), p(b2), p(scale), p(bias), p(gate), p(x_out), p(a_out),
                                                  b, l, c, h, _stream(y)), "mjx_nn_block_tail_bf16")
    return x_out, a_out


def post_block_tail(y: torch.Tensor, x: torch.Tensor, scale: torch.Tensor, bias: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor,
                    w2t: torch.Tensor, b2: torch.Tensor) -> torch.Tensor:
    """The post-activation block's tail (version 1): t = y * scale + bias (its second BatchNorm), gate = sigmoid(mlp(mean_L t) +
    mlp(max_L t)) with mlp(v) = w2 @ relu(w1 @ v + b1) + b2 (float32: w1 [H, C], w2t = w2.T [H, C]); returns relu(t * gate + x)."""
    b, c, l = _check_nhwc(y)
    assert _check_nhwc(x) == (b, c, l)
    h = w1.shape[0]
    for t, shape in ((scale, (c,)), (bias, (c,)), (w1, (h, c)), (b1, (h,)), (w2t, (h, c)), (b2, (c,))):
        assert t.dtype == torch.float32 and tuple(t.shape) == shape and t.is_contiguous() and t.is_cuda
    _aligned(scale, bias, w1, b1, w2t, b2)
    assert c <= 256, "post_block_tail: at most 256 channels"
    x_out = torch.empty_like(y)
    gate = torch.empty((b, c), dtype=torch.bfloat16, device=y.device)
    p = lambda t: C.c_void_p(t.data_ptr())
    _lib.check(_lib.load().mjx_nn_post_block_tail_bf16(p(y), p(x), p(scale), p(bias), p(w1), p(b1), p(w2t), p(b2), p(gate), p(x_out),
                                                       b, l, c, h, _stream(y)), "mjx_nn_post_block_tail_bf16")
    return x_out


def obs_to_nhwc(obs: torch.Tensor, channels_padded: int) -> torch.Tensor:
    """f32 [B, C, L] (contiguous) -> bf16 [B, channels_padded, 1, L] in channels_last memory format, extra channels zero."""
    assert obs.is_cuda and obs.dtype == torch.float32 and obs.dim() == 3 and obs.is_contiguous()
    b, c, l = obs.shape
    assert channels_padded >= c and channels_padded % 64 == 0
    out = torch.empty((b, channels_padded, 1, l), dtype=torch.bfloat16, device=obs.device, memory_format=torch.channels_last)
    _lib.check(_lib.load().mjx_nn_obs_to_nhwc_bf16(C.c_void_p(obs.data_ptr()), C.c_void_p(out.data_ptr()), b, c, l, channels_padded,
                                                   _stream(obs)), "mjx_nn_obs_to_nhwc_bf16")
    return out


def obs2_to_nhwc(obs: torch.Tensor, obs2: torch.Tensor, channels_padded: int) -> torch.Tensor:
    """The input of an oracle brain's stem: f32 obs [B, C1, L] and invisible obs [B, C2, L] (contiguous) -> bf16
    [B, channels_padded, 1, L] channels_last holding obs's channels, then obs2's, then zeros (torch.cat((obs, obs2), 1), padded)."""
    for t in (obs, obs2):
        assert t.is_cuda and t.dtype == torch.float32 and t.dim() == 3 and t.is_contiguous()
    b, c1, l = obs.shape
    c2 = obs2.shape[1]
    assert obs2.shape == (b, c2, l) and obs2.device == obs.device
    assert channels_padded >= c1 + c2 and channels_padded % 64 == 0
    out = torch.empty((b, channels_padded, 1, l), dtype=torch.bfloat16, device=obs.device, memory_format=torch.channels_last)
    _lib.check(_lib.load().mjx_nn_obs2_to_nhwc_bf16(C.c_void_p(obs.data_ptr()), C.c_void_p(obs2.data_ptr()), C.c_void_p(out.data_ptr()),
                                                    b, c1, c2, l, channels_padded, _stream(obs)), "mjx_nn_obs2_to_nhwc_bf16")
    return out
