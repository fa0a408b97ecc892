"""ctypes wrappers and autograd Functions of the fused policy-net training kernels in libmjx (csrc/mjx_train.cuh).

Activations are CUDA tensors logically [B, C, 1, L] in channels_last memory format ([B, L, C] in memory), float32 (a run without
AMP) or float16 (under `torch.autocast('cuda')`, whose default dtype is float16), with 1 <= C <= 256 and C % 8 == 0. The kernels
compute in float32 and reduce in an order fixed by the shape, so two calls on the same inputs give bit-identical results.

- `bn_mish(x, bn, frozen, group)`: BatchNorm1d + Mish of a pre-activation, train mode (batch statistics, running statistics updated
  as nn.BatchNorm1d updates them) or frozen (running statistics, untouched). With a torch.distributed `group` of more than one
  rank, train mode uses the statistics of the batch all the group's ranks hold together (synchronised BatchNorm).
- `gate_residual(y, x, gate)`: ChannelGate(y) + x, the gate's shared MLP in torch (float32) on the pooled [B, C] vectors.
- `dqn_losses(...)`: mortal/train.py:228-247 over the dueling head's v / a and the aux logits, in one launch.
"""
from __future__ import annotations

import ctypes as C
import os

import torch
import torch.nn.functional as F

from . import _cdecl, _lib

HEADER = os.path.join(os.path.dirname(_cdecl.HEADER), "mjx_train_ranks.h")
with open(HEADER) as _f:
    SYMBOLS = _cdecl.functions(_f.read(), "mjx_")  # the entries of include/mjx_train_ranks.h, exported by libmjx.so
_RANKS = None


def ranks_lib():
    """libmjx.so with the data-parallel BatchNorm entries of include/mjx_train_ranks.h bound"""
    global _RANKS
    if _RANKS is None:
        _RANKS = _cdecl.bind(_lib.load(), SYMBOLS)
    return _RANKS

_DTYPES = {torch.float32: 0, torch.float16: 1}


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _stream(t: torch.Tensor):
    return C.c_void_p(torch._C._cuda_getCurrentRawStream(t.device.index))


def _dtype_code(t: torch.Tensor) -> int:
    if t.dtype not in _DTYPES:
        raise ValueError(f"train_ops: activations must be float32 or float16, got {t.dtype}")
    return _DTYPES[t.dtype]


def check_channels(c: int):
    if c <= 0 or c > 256 or c % 8:
        raise ValueError(f"the fused training kernels take a channel count that is a multiple of 8, at most 256; got {c}")


def _nhwc(x: torch.Tensor):
    """[B, C, 1, L] -> its channels_last contiguous form and (B, C, L); ValueError for any other shape"""
    if not x.is_cuda or x.dim() != 4 or x.shape[2] != 1 or x.shape[0] < 1:
        raise ValueError(f"train_ops: expected a CUDA tensor [B >= 1, C, 1, L], got {tuple(x.shape)} on {x.device}")
    b, c, _, l = x.shape
    check_channels(c)
    _dtype_code(x)
    if b * l * c >= 1 << 31:
        raise ValueError(f"train_ops: at most 2^31 - 1 activations per tensor, got {b} x {c} x {l}")
    return x.contiguous(memory_format=torch.channels_last), b, c, l


_SCRATCH = {}


def _scratch_floats(rows: int, c: int) -> int:
    key = (rows, c)
    if key not in _SCRATCH:
        _SCRATCH[key] = _lib.load().mjx_train_bn_scratch_floats(rows, c)
    return _SCRATCH[key]


class _BatchNormMish(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, eps, momentum, training, group):
        x, b, c, l = _nhwc(x)
        out = torch.empty_like(x)
        stats = torch.empty(3 * c, dtype=torch.float32, device=x.device)
        mean, invstd = stats[: 2 * c], stats[2 * c:]  # the batch mean as a float pair (hi, lo), and 1 / sqrt(var + eps)
        L = _lib.load()
        scratch = torch.empty(_scratch_floats(b * l, c), dtype=torch.float32, device=x.device)
        if group is None:
            _lib.check(L.mjx_train_bn_mish_fwd(_dtype_code(x), _p(x), _p(weight), _p(bias), _p(running_mean), _p(running_var),
                                               _p(mean), _p(invstd), _p(out), b * l, c, float(eps), float(momentum), int(training),
                                               _p(scratch), _stream(x)), "mjx_train_bn_mish_fwd")
        else:
            import torch.distributed as dist

            L = ranks_lib()
            rank, world = dist.get_rank(group), dist.get_world_size(group)
            rows = torch.zeros((world, 3, c), dtype=torch.float64, device=x.device)  # (count, mean, M2) per rank
            _lib.check(L.mjx_train_bn_local_stats(_dtype_code(x), _p(x), b * l, c, rank, world, _p(rows), _p(scratch), _stream(x)),
                       "mjx_train_bn_local_stats")
            # each rank wrote its own row into zeros: the SUM adds exact zeros, so this is a bit-exact all-gather (one that gloo
            # also runs on CUDA tensors) and every rank merges the same rows
            dist.all_reduce(rows, group=group)
            _lib.check(L.mjx_train_bn_mish_fwd_ranks(_dtype_code(x), _p(x), _p(weight), _p(bias), _p(running_mean), _p(running_var),
                                                     _p(mean), _p(invstd), _p(out), b * l, c, float(eps), float(momentum), _p(rows),
                                                     world, _stream(x)), "mjx_train_bn_mish_fwd_ranks")
        ctx.save_for_backward(x, weight, bias, mean, invstd)
        ctx.training, ctx.group = bool(training), group
        return out

    @staticmethod
    def backward(ctx, dout):
        x, weight, bias, mean, invstd = ctx.saved_tensors
        b, c, _, l = x.shape
        dout = dout.to(x.dtype).contiguous(memory_format=torch.channels_last)
        dx = torch.empty_like(x)
        dgamma = torch.empty(c, dtype=torch.float32, device=x.device)
        dbeta = torch.empty_like(dgamma)
        L = _lib.load()
        scratch = torch.empty(_scratch_floats(b * l, c), dtype=torch.float32, device=x.device)
        code, group = _dtype_code(x), ctx.group
        if group is None:
            _lib.check(L.mjx_train_bn_mish_bwd(code, _p(x), _p(dout), _p(weight), _p(bias), _p(mean), _p(invstd), _p(dx), _p(dgamma),
                                               _p(dbeta), b * l, c, int(ctx.training), _p(scratch), _stream(x)), "mjx_train_bn_mish_bwd")
        else:
            import torch.distributed as dist

            L = ranks_lib()
            rank, world = dist.get_rank(group), dist.get_world_size(group)
            sums = torch.zeros((world, 2, c), dtype=torch.float64, device=x.device)  # (sum dz, sum dz xhat) per rank
            _lib.check(L.mjx_train_bn_bwd_local_sums(code, _p(x), _p(dout), _p(weight), _p(bias), _p(mean), _p(invstd), b * l, c, rank,
                                                     world, _p(sums), _p(scratch), _stream(x)), "mjx_train_bn_bwd_local_sums")
            dist.all_reduce(sums, group=group)  # the bit-exact all-gather of the forward's rows
            # every rank holds b * l rows (bn_mish's condition); dgamma / dbeta are this rank's share
            _lib.check(L.mjx_train_bn_mish_bwd_ranks(code, _p(x), _p(dout), _p(weight), _p(bias), _p(mean), _p(invstd), _p(dx),
                                                     _p(dgamma), _p(dbeta), b * l, c, _p(sums), rank, world, world * b * l, _p(scratch),
                                                     _stream(x)), "mjx_train_bn_mish_bwd_ranks")
        return dx, dgamma.to(weight.dtype), dbeta.to(bias.dtype), None, None, None, None, None, None


def bn_mish(x: torch.Tensor, bn: torch.nn.BatchNorm1d, frozen: bool = False, group=None) -> torch.Tensor:
    """mish(bn(x)) for x [B, C, 1, L] channels_last. Unless `frozen` or `bn` is in eval mode, the batch statistics are used and
    bn's running_mean / running_var / num_batches_tracked are updated as nn.BatchNorm1d.forward in train mode updates them.

    `group`: a torch.distributed process group whose every rank calls this with an x of the same shape, as data-parallel ranks
    do. With more than one rank, training mode normalises with the statistics of all the ranks' rows together (exchanged twice
    per forward and backward, in double), which every rank computes bit for bit alike, so the running statistics stay equal;
    the parameter gradients are this rank's share, for the caller's gradient all-reduce to sum or average. None (or one rank):
    this process's rows alone."""
    training = bn.training and not frozen
    if group is not None:
        import torch.distributed as dist

        world = dist.get_world_size(group)
        if world == 1 or not training:  # one rank, or the running statistics: nothing to exchange
            group = None
    else:
        world = 1
    if training and bn.momentum is None:
        raise ValueError("bn_mish: a cumulative moving average (momentum=None) is not supported")
    if training and world * x.shape[0] * x.shape[3] < 2:
        raise ValueError("bn_mish: training-mode BatchNorm needs more than one value per channel")
    for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var):
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError("bn_mish: the BatchNorm's parameters and statistics must be contiguous float32")
    out = _BatchNormMish.apply(x, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps, bn.momentum or 0.0, training, group)
    if training:
        bn.num_batches_tracked.add_(1)
    return out


def _gate_mlp(v, w1, b1, w2, b2):
    """the shared MLP on the concatenated pooled vectors v = [avg; max] ([2B, C], float32): (pre-activation of the hidden layer,
    gate = sigmoid(mlp(avg) + mlp(max)))"""
    h1 = F.linear(v, w1, b1)
    h2 = F.linear(F.mish(h1), w2, b2)
    b = v.shape[0] // 2
    return h1, torch.sigmoid(h2[:b] + h2[b:])


class _GateResidual(torch.autograd.Function):
    """ChannelGate(y) + x. The gate MLP runs on [2B, C] vectors in float32 (also under autocast: it is tiny, and float32 keeps its
    hand-written backward exact), its backward in closed form: no autograd graph is recorded or replayed per block."""

    @staticmethod
    def forward(ctx, y, x, w1, b1, w2, b2):
        y, b, c, l = _nhwc(y)
        x = x.to(y.dtype).contiguous(memory_format=torch.channels_last)
        code, L = _dtype_code(y), _lib.load()
        avg = torch.empty((2 * b, c), dtype=y.dtype, device=y.device)  # [avg; max]
        _lib.check(L.mjx_train_gate_pool(code, _p(y), _p(avg[:b]), _p(avg[b:]), b, l, c, _stream(y)), "mjx_train_gate_pool")
        with torch.autocast("cuda", enabled=False):
            v = avg.float()
            h1, g = _gate_mlp(v, w1.float(), b1.float(), w2.float(), b2.float())
        gt = g.to(y.dtype)
        out = torch.empty_like(y)
        _lib.check(L.mjx_train_gate_out(code, _p(y), _p(gt), _p(x), _p(out), b, l, c, _stream(y)), "mjx_train_gate_out")
        ctx.save_for_backward(y, avg, v, h1, g, gt, w1, w2)
        return out

    @staticmethod
    def backward(ctx, dout):
        y, avg, v, h1, g, gt, w1, w2 = ctx.saved_tensors
        b, c, _, l = y.shape
        code, L = _dtype_code(y), _lib.load()
        dout = dout.to(y.dtype).contiguous(memory_format=torch.channels_last)
        dg = torch.empty((b, c), dtype=torch.float32, device=y.device)
        cnt = torch.empty((b, c), dtype=torch.float32, device=y.device)
        _lib.check(L.mjx_train_gate_bwd_dg(code, _p(dout), _p(y), _p(avg[b:]), _p(dg), _p(cnt), b, l, c, _stream(y)),
                   "mjx_train_gate_bwd_dg")
        with torch.autocast("cuda", enabled=False):
            ds = dg * g * (1 - g)                      # through the sigmoid; the same gradient reaches both MLP passes
            dh2 = torch.cat((ds, ds), 0)
            a1 = F.mish(h1)
            dw2, db2 = dh2.t().mm(a1), 2 * ds.sum(0)
            dh1 = torch.ops.aten.mish_backward(dh2.mm(w2.float()), h1)
            dw1, db1 = dh1.t().mm(v), dh1.sum(0)
            dv = dh1.mm(w1.float()).to(y.dtype)     # [d_avg; d_max]
        dy = torch.empty_like(y)
        _lib.check(L.mjx_train_gate_bwd_dy(code, _p(dout), _p(y), _p(gt), _p(avg[b:]), _p(cnt), _p(dv[:b]), _p(dv[b:]), _p(dy), b, l, c,
                                           _stream(y)), "mjx_train_gate_bwd_dy")
        return dy, dout, dw1, db1, dw2, db2


def gate_residual(y: torch.Tensor, x: torch.Tensor, gate) -> torch.Tensor:
    """gate(y) + x for y, x [B, C, 1, L] channels_last and `gate` a model.ChannelGate with a Mish hidden layer"""
    return _GateResidual.apply(y, x, gate.fc1.weight, gate.fc1.bias, gate.fc2.weight, gate.fc2.bias)


class _DqnLosses(torch.autograd.Function):
    @staticmethod
    def forward(ctx, v, a, aux, masks, actions, steps_to_done, kyoku_rewards, player_ranks, gamma):
        b = v.shape[0]
        n_aux = aux.shape[1]
        code, L = _dtype_code(v), _lib.load()
        dev = v.device
        q = torch.empty(b, dtype=torch.float32, device=dev)
        q_target = torch.empty_like(q)
        losses = torch.empty(3, dtype=torch.float32, device=dev)
        bad = torch.zeros((), dtype=torch.int32, device=dev)
        _lib.check(L.mjx_train_dqn_loss_fwd(code, _p(v), _p(a), _p(masks), _p(actions), _p(steps_to_done), _p(kyoku_rewards), _p(aux),
                                            _p(player_ranks), b, n_aux, float(gamma), C.c_void_p(0), _p(q), _p(q_target), _p(losses),
                                            _p(bad), _stream(v)), "mjx_train_dqn_loss_fwd")
        ctx.save_for_backward(v, a, aux, masks, actions, q_target, player_ranks)
        ctx.mark_non_differentiable(q, q_target, bad)
        return losses[0], losses[1], losses[2], q, q_target, bad

    @staticmethod
    def backward(ctx, g_dqn, g_cql, g_rank, *_):
        v, a, aux, masks, actions, q_target, player_ranks = ctx.saved_tensors
        b, n_aux = v.shape[0], aux.shape[1]
        zero = torch.zeros((), dtype=torch.float32, device=v.device)
        w = torch.stack([zero if g is None else g.float().reshape(()) for g in (g_dqn, g_cql, g_rank)]).contiguous()
        dv, da, daux = torch.empty_like(v), torch.empty_like(a), torch.empty_like(aux)
        _lib.check(_lib.load().mjx_train_dqn_loss_bwd(_dtype_code(v), _p(v), _p(a), _p(masks), _p(actions), _p(q_target), _p(aux),
                                                      _p(player_ranks), b, n_aux, _p(w), _p(dv), _p(da), _p(daux), _stream(v)),
                   "mjx_train_dqn_loss_bwd")
        return dv, da, daux, None, None, None, None, None, None


def dqn_losses(v, a, aux_logits, masks, actions, steps_to_done, kyoku_rewards, player_ranks, gamma):
    """mortal/train.py:228-247 in one launch: the masked dueling combine q_out = v + a - mean_legal(a) (-inf off the mask),
    q = q_out[i, actions], q_target = (gamma ** steps_to_done * kyoku_rewards).float(), and
    (dqn_loss = 0.5 mse(q, q_target), cql_loss = mean logsumexp(q_out) - mean q, next_rank_loss = cross_entropy(aux_logits,
    player_ranks), q, q_target, bad). v [B, 1], a [B, 46], aux_logits [B, n] (float32 or float16, one dtype); masks bool [B, 46];
    actions / steps_to_done / player_ranks int64 [B]; kyoku_rewards float64 [B]. The three losses are differentiable with respect
    to v, a and aux_logits; `bad` is an int32 device scalar, nonzero when an action lies outside its mask (no host sync)."""
    b = v.shape[0]
    if b < 1 or v.shape != (b, 1) or a.shape != (b, 46) or aux_logits.dim() != 2 or aux_logits.shape[0] != b or not 1 <= aux_logits.shape[1] <= 32:
        raise ValueError(f"dqn_losses: expected v [B, 1], a [B, 46], aux_logits [B, n <= 32]; got {tuple(v.shape)}, {tuple(a.shape)}, "
                         f"{tuple(aux_logits.shape)}")
    if masks.shape != (b, 46) or masks.dtype != torch.bool:
        raise ValueError("dqn_losses: masks must be bool [B, 46]")
    _dtype_code(v)
    a, aux_logits = a.to(v.dtype), aux_logits.to(v.dtype)
    cols = [actions, steps_to_done, player_ranks]
    if any(t.shape != (b,) or t.dtype != torch.int64 for t in cols) or kyoku_rewards.shape != (b,) or kyoku_rewards.dtype != torch.float64:
        raise ValueError("dqn_losses: actions / steps_to_done / player_ranks must be int64 [B] and kyoku_rewards float64 [B]")
    return _DqnLosses.apply(v.contiguous(), a.contiguous(), aux_logits.contiguous(), masks.contiguous().view(torch.uint8),
                            actions.contiguous(), steps_to_done.contiguous(), kyoku_rewards.contiguous(), player_ranks.contiguous(),
                            float(gamma))
