"""float64 references and error bounds for the fused policy-net kernels (mortal_b200/csrc/mjx_nn.cuh) and the cuDNN (1 x 3)
convolutions between them.

Every reference takes the kernel's actual inputs (bf16 activations, fp32 parameters) and computes the operation in float64, so
what is left between a kernel's output and the reference is the kernel's own arithmetic and the final rounding to bf16. Each
bound below says how much of that a correct kernel may show; a future kernel for the same op is held to the same function.

Layouts follow the kernels: activations are logically [B, C, 1, L] (channels_last in memory), pooled vectors and gates [B, C].
All functions work on CPU and CUDA tensors alike.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

F64 = torch.float64
NHWC_DIMS = ("b", "c", "_", "l")  # index names of a [B, C, 1, L] activation, for failure messages
BC_DIMS = ("b", "c")


def f64(t: torch.Tensor) -> torch.Tensor:
    return t.to(F64)  # bf16 / fp32 -> float64 is exact


def rn_bf16(v: torch.Tensor) -> torch.Tensor:
    """float64 -> fp32 -> bf16, each round-to-nearest-even: what a kernel's fp32 result followed by __float2bfloat16_rn is."""
    return v.to(torch.float32).to(torch.bfloat16)


# ---- bf16 spacing ------------------------------------------------------------------------------------------------------

def ulp_bf16(v: torch.Tensor) -> torch.Tensor:
    """The spacing of bf16 numbers in the binade of |v| (float64): 2^(floor(log2 |v|) - 7) for normal |v|, 2^-133 for subnormal
    |v| and 0. For a bf16 value x this is nextafter(x, +inf) - x (x > 0); rounding v to nearest errs by at most half of it."""
    a = f64(v).abs()
    _, e = torch.frexp(a)  # a = m 2^e, m in [0.5, 1): floor(log2 a) = e - 1 (exact, unlike log2 just below a power of two)
    e = torch.where(a == 0, torch.full_like(e, -126), (e - 1).clamp(min=-126))
    return torch.ldexp(torch.ones_like(a), e - 7)


def half_ulp_bf16(v: torch.Tensor) -> torch.Tensor:
    return ulp_bf16(v) * 0.5


# ---- the per-op references (float64) ----------------------------------------------------------------------------------

def _cvec(p: torch.Tensor, like: torch.Tensor) -> torch.Tensor:
    return f64(p).view(1, -1, *([1] * (like.dim() - 2)))


def pre_activation(x: torch.Tensor, scale: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """t = x * scale[c] + bias[c] (the eval-mode BatchNorm as an affine) in float64; x [B, C, ...]"""
    return f64(x) * _cvec(scale, x) + _cvec(bias, x)


def mish(t: torch.Tensor) -> torch.Tensor:
    """x tanh(softplus(x)) in float64; -inf -> NaN, +inf -> +inf, NaN -> NaN"""
    return F.mish(f64(t))


def affine_mish(x: torch.Tensor, scale: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """mish(x * scale[c] + bias[c]). The pre-activation is an fp32 value by contract: where it lies beyond the fp32 range
    (bf16-max x 2) it is taken as the ±inf fp32 makes of it, so a pre-activation below -FLT_MAX gives NaN, not -0."""
    t = pre_activation(x, scale, bias)
    t32 = t.to(torch.float32)
    return mish(torch.where(torch.isinf(t32) & torch.isfinite(t), f64(t32), t))


def pool_mean_max(y: torch.Tensor):
    """(mean over L, max over L) of [B, C, 1, L] -> two float64 [B, C]. The max propagates NaN (torch.amax)."""
    y = f64(y).flatten(2)
    return y.mean(-1), y.amax(-1)


def gate(y: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor, w2t: torch.Tensor, b2: torch.Tensor):
    """The channel gate of [B, C, 1, L] y: sigmoid(mlp(mean_L y) + mlp(max_L y)), mlp(v) = w2 mish(w1 v + b1) + b2
    (w1 [H, C], w2t = w2^T [H, C], fp32). Returns (g, zabs), both float64 [B, C]: zabs is the logit z recomputed with every
    term replaced by its absolute value (|mish(p)| <= |p|), the scale of the rounding error a float32 evaluation can make."""
    w1, b1, w2t, b2 = f64(w1), f64(b1), f64(w2t), f64(b2)
    z = zabs = 0
    for v in pool_mean_max(y):
        z = z + mish(v @ w1.T + b1) @ w2t + b2
        zabs = zabs + ((v.abs() @ w1.abs().T + b1.abs()) @ w2t.abs() + b2.abs())
    return torch.sigmoid(z), zabs


def gate_residual(y: torch.Tensor, g: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """y * g[b, c] + x in float64 ([B, C, 1, L], g [B, C]). With bf16 y and g the product is exact, so rn_bf16 of this is the
    kernel's fmaf (one rounding to fp32) followed by the rounding to bf16."""
    return f64(y) * f64(g).view(g.shape[0], g.shape[1], 1, 1) + f64(x)


def stem_input(obs: torch.Tensor, channels_padded: int) -> torch.Tensor:
    """The stem transform: observations [B, C, L] -> [B, channels_padded, 1, L] float64, extra channels zero."""
    b, c, l = obs.shape
    out = torch.zeros((b, channels_padded, 1, l), dtype=F64, device=obs.device)
    out[:, :c, 0] = f64(obs)
    return out


def conv1x3(a: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None):
    """The (1 x 3) convolution with padding 1 of a [B, Cin, 1, L] by w [Cout, Cin, 1, 3] (or a Conv1d's [Cout, Cin, 3]) in float64,
    as a matrix product of the unfolded input. Returns (v, s), both [B, Cout, 1, L]: the result and sum |w a| (+ |bias|)."""
    a = f64(a).squeeze(2)
    b, cin, l = a.shape
    w = f64(w).reshape(w.shape[0], cin * 3)
    ap = F.pad(a, (1, 1))
    cols = torch.stack([ap[..., k:k + l] for k in range(3)], dim=-1)  # [B, Cin, L, 3]
    cols = cols.permute(0, 2, 1, 3).reshape(b * l, cin * 3)
    v, s = cols @ w.T, cols.abs() @ w.abs().T
    if bias is not None:
        v, s = v + f64(bias), s + f64(bias).abs()
    shape = lambda t: t.view(b, l, -1).permute(0, 2, 1).unsqueeze(2)
    return shape(v), shape(s)


# ---- bounds: |got - v| <= bound(...) for a kernel output `got` (bf16) and the float64 value v of the same inputs -------------

def bound_affine_mish(v: torch.Tensor) -> torch.Tensor:
    """mish(x * scale + bias): half an ulp for the rounding to bf16, 2^-16 |v| for the fp32 FMA, SFU exp and reciprocal
    (about (2 |t| + 8) 2^-24 relative for a pre-activation |t| up to ~100), and 2^-110 absolute: below t ~ -87 the exponential
    flushes to zero, so results that small may come out as (-)0."""
    v = f64(v)
    return half_ulp_bf16(v) + 2.0 ** -16 * v.abs() + 2.0 ** -110


def bound_pool_max(v: torch.Tensor) -> torch.Tensor:
    """The max of bf16 values is a bf16 value: bit-exact."""
    return torch.zeros_like(f64(v))


def bound_pool_mean(v: torch.Tensor, mean_abs: torch.Tensor, length: int) -> torch.Tensor:
    """The mean as an fp32 running sum times fp32 1/L: L - 1 rounded additions, the rounded 1/L and the product each cost
    2^-24 mean|x| at most, plus half an ulp for the rounding to bf16."""
    return half_ulp_bf16(v) + (length + 1) * 2.0 ** -24 * f64(mean_abs)


def bound_gate(g: torch.Tensor, zabs: torch.Tensor, length: int, channels: int, hidden: int) -> torch.Tensor:
    """The gate (fp32 logit z -> sigmoid -> bf16): an error dz in z moves g by g (1 - g) dz. dz = (L + C + H) 2^-23 zabs covers
    the pooling, the two dot products and the hidden Mish in fp32; 2^-21 the SFU exp of the sigmoid ((2 + 1.2 |z|) ulp); 2^-23 g
    the rounding of 1 + e and of the reciprocal; 2^-110 an exponential that overflows for z below ~ -88; half an ulp the bf16."""
    g = f64(g)
    dz = (length + channels + hidden) * 2.0 ** -23 * f64(zabs) + 2.0 ** -21
    return half_ulp_bf16(g) + g * (1 - g) * dz + 2.0 ** -23 * g + 2.0 ** -110


def bound_conv(v: torch.Tensor, sum_abs: torch.Tensor, cin: int, unbiased: torch.Tensor | None = None) -> torch.Tensor:
    """A (1 x 3) convolution with bf16 inputs, fp32 accumulation and bf16 output: K = 3 Cin products accumulated at 2^-22 each
    relative to sum |w a| (not a proven bound for the tensor cores: the GPU test measures how much of it is used), plus half an
    ulp for the output rounding. With a bias, PyTorch rounds the product sum to bf16 before it adds the bias: pass that
    unbiased value to allow its half ulp as well."""
    b = half_ulp_bf16(v) + 3 * cin * 2.0 ** -22 * f64(sum_abs)
    return b if unbiased is None else b + half_ulp_bf16(unbiased)


# ---- checkers: the worst element, by name ----------------------------------------------------------------------------------

def _where(flat: int, shape, dims) -> str:
    idx = []
    for n in reversed(shape):
        idx.append(flat % n)
        flat //= n
    idx = idx[::-1]
    names = dims if dims is not None and len(dims) == len(shape) else [f"d{i}" for i in range(len(shape))]
    return ", ".join(f"{k}={i}" for k, i in zip(names, idx) if k != "_")


def worst_violation(got: torch.Tensor, v: torch.Tensor, bound: torch.Tensor, dims=None):
    """(excess, where, got, v, bound) of the element where |got - v| - bound is largest. Where got or the correctly rounded v is
    not finite, the two must be equal (NaN matches NaN): excess is -inf if they are and +inf if not. excess <= 0: all within."""
    g, v, bound = f64(got), f64(v), f64(bound).expand_as(f64(v))
    rv = f64(rn_bf16(v))
    excess = (g - v).abs() - bound
    nonfinite = ~torch.isfinite(g) | ~torch.isfinite(rv)
    same = (torch.isnan(g) & torch.isnan(rv)) | (g == rv)
    inf = torch.full_like(excess, float("inf"))
    excess = torch.where(nonfinite, torch.where(same, -inf, inf), excess)
    i = int(torch.argmax(excess.flatten()))
    return (excess.flatten()[i].item(), _where(i, tuple(v.shape), dims), g.flatten()[i].item(), v.flatten()[i].item(),
            bound.flatten()[i].item())


def check_within(what: str, got: torch.Tensor, v: torch.Tensor, bound: torch.Tensor, dims=None):
    assert got.shape == v.shape, (what, tuple(got.shape), tuple(v.shape))
    excess, where, g, vv, b = worst_violation(got, v, bound, dims)
    assert excess <= 0, f"{what}: |got - v| exceeds its bound by {excess:.3g} at {where}: got {g!r}, v {vv!r}, bound {b:.3g}"


def check_bits(what: str, got: torch.Tensor, ref: torch.Tensor, dims=None):
    """bf16 bit for bit; NaN is compared by NaN-ness, zero by sign."""
    assert got.dtype == ref.dtype == torch.bfloat16 and got.shape == ref.shape, (what, got.dtype, ref.dtype, got.shape, ref.shape)
    g, r = got.contiguous(), ref.contiguous()
    bad = (g.view(torch.int16) != r.view(torch.int16)) & ~(torch.isnan(g) & torch.isnan(r))
    if bad.any():
        i = int(torch.nonzero(bad.flatten())[0])
        raise AssertionError(f"{what}: {int(bad.sum())} values differ, first at {_where(i, tuple(g.shape), dims)}: "
                             f"got {g.flatten()[i].item()!r}, expected {r.flatten()[i].item()!r}")
