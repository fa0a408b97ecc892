"""Policy/value networks of every Mortal version, as ordinary PyTorch modules, and the loader of Mortal checkpoints.

Architectures restated from mortal/model.py:10-231. Versions 2-4: Conv1d stem -> `num_blocks` pre-activation residual blocks
(BN -> Mish -> Conv1d k3, twice) each gated by a squeeze/excite style channel attention (Mish hidden layer) -> BN -> Mish ->
Conv1d(C, 32, k3) -> Mish -> Linear(32*34, 1024) -> Mish. Version 1: Conv1d stem -> BN -> ReLU -> `num_blocks` post-activation
blocks (Conv1d -> BN -> ReLU -> Conv1d -> BN -> attention with a ReLU hidden layer -> + x -> ReLU) -> Conv1d(C, 32, k3) -> ReLU ->
Linear(32*34, 1024) -> latent Linear(1024, 512) + ReLU -> mu / logsig heads. Oracle brains read the observation and the invisible
observation concatenated along the channels. DQN heads: version 4 Linear(1024, 1+46); versions 2 / 3 two Linear-Mish-Linear
heads (hidden 512 / 256); version 1 Linear heads on the 512-wide latent; the advantage mean is taken over legal actions only and
illegal actions are -inf.

The modules use their own parameter names; `load_mortal` is the one place that knows the reference's checkpoint key layout.
"""
from __future__ import annotations

import re

import torch
from torch import nn

OBS_ROWS = {1: 938, 2: 942, 3: 934, 4: 1012}  # consts.rs:20-28
ORACLE_ROWS = {1: 211, 2: 217, 3: 217, 4: 217}  # consts.rs oracle_obs_shape
BN_EPS = {1: 1e-5, 2: 1e-5, 3: 1e-3, 4: 1e-3}  # not stored in a checkpoint: it follows from the version
ACTION_SPACE = 46


class ChannelGate(nn.Module):
    def __init__(self, channels: int, ratio: int = 16, act=nn.Mish):
        super().__init__()
        self.fc1 = nn.Linear(channels, channels // ratio)
        self.fc2 = nn.Linear(channels // ratio, channels)
        nn.init.zeros_(self.fc1.bias)
        nn.init.zeros_(self.fc2.bias)
        self.act = act(inplace=True)

    def _mlp(self, v):
        return self.fc2(self.act(self.fc1(v)))

    def forward(self, x):
        gate = torch.sigmoid(self._mlp(x.mean(-1)) + self._mlp(x.amax(-1)))
        return x * gate.unsqueeze(-1)

    def forward_fast(self, x):
        # x: [B, C, 1, L] channels_last; same maths as forward()
        gate = torch.sigmoid(self._mlp(x.mean((2, 3))) + self._mlp(x.amax((2, 3))))
        return x * gate.view(gate.shape[0], gate.shape[1], 1, 1)


class PreActBlock(nn.Module):
    def __init__(self, channels: int, eps: float = 1e-3):
        super().__init__()
        self.bn1 = nn.BatchNorm1d(channels, momentum=0.01, eps=eps)
        self.conv1 = nn.Conv1d(channels, channels, 3, padding=1, bias=False)
        self.bn2 = nn.BatchNorm1d(channels, momentum=0.01, eps=eps)
        self.conv2 = nn.Conv1d(channels, channels, 3, padding=1, bias=False)
        self.act = nn.Mish(inplace=True)
        self.gate = ChannelGate(channels)

    def forward(self, x):
        y = self.conv1(self.act(self.bn1(x)))
        y = self.conv2(self.act(self.bn2(y)))
        return self.gate(y) + x

    @staticmethod
    def _affine(bn):
        # eval-mode BatchNorm is a per-channel affine map: y = x * scale + shift
        scale = bn.weight / torch.sqrt(bn.running_var + bn.eps)
        shift = bn.bias - bn.running_mean * scale
        return scale.view(1, -1, 1, 1).contiguous(), shift.view(1, -1, 1, 1).contiguous()

    def forward_fast(self, x, aff, w1, w2, aff32=None):
        (s1, b1), (s2, b2) = aff
        F = torch.nn.functional
        if aff32 is not None and x.is_cuda and x.dtype == torch.bfloat16:
            # fused bandwidth-bound passes (libmjx, csrc/mjx_nn.cuh) around the two cuDNN convolutions
            from . import nn_ops

            (f1, g1), (f2, g2) = aff32
            y = F.conv2d(nn_ops.affine_mish(x, f1, g1), w1, padding=(0, 1))
            y = F.conv2d(nn_ops.affine_mish(y, f2, g2), w2, padding=(0, 1))
            avg, mx = nn_ops.pool_mean_max(y)
            h = self.gate._mlp(torch.cat((avg, mx), 0))  # both pooled vectors through the gate MLP in one call
            gate = torch.sigmoid(h[: avg.shape[0]] + h[avg.shape[0]:])
            return nn_ops.gate_residual(y, gate.contiguous(), x)
        y = F.conv2d(F.mish(torch.addcmul(b1, x, s1)), w1, padding=(0, 1))
        y = F.conv2d(F.mish(torch.addcmul(b2, y, s2)), w2, padding=(0, 1))
        return self.gate.forward_fast(y) + x


class PostActBlock(nn.Module):
    """Version 1's residual block (mortal/model.py ResBlock with pre_actv=False)."""

    def __init__(self, channels: int, eps: float = 1e-5):
        super().__init__()
        self.conv1 = nn.Conv1d(channels, channels, 3, padding=1, bias=False)
        self.bn1 = nn.BatchNorm1d(channels, momentum=0.01, eps=eps)
        self.conv2 = nn.Conv1d(channels, channels, 3, padding=1, bias=False)
        self.bn2 = nn.BatchNorm1d(channels, momentum=0.01, eps=eps)
        self.act = nn.ReLU(inplace=True)
        self.gate = ChannelGate(channels, act=nn.ReLU)

    def forward(self, x):
        y = self.act(self.bn1(self.conv1(x)))
        y = self.bn2(self.conv2(y))
        return self.act(self.gate(y) + x)

    def forward_fast(self, x, aff, w1, w2):
        (s1, b1), (s2, b2) = aff
        F = torch.nn.functional
        y = F.relu(torch.addcmul(b1, F.conv2d(x, w1, padding=(0, 1)), s1))
        y = torch.addcmul(b2, F.conv2d(y, w2, padding=(0, 1)), s2)
        return F.relu(self.gate.forward_fast(y) + x)


class Brain(nn.Module):
    def __init__(self, *, conv_channels: int = 192, num_blocks: int = 40, version: int = 4, is_oracle: bool = False):
        super().__init__()
        if version not in OBS_ROWS:
            raise ValueError(f"unsupported Mortal version {version!r} (1..4)")
        self.version, self.is_oracle = version, bool(is_oracle)
        c, eps = conv_channels, BN_EPS[version]
        self.stem = nn.Conv1d(OBS_ROWS[version] + (ORACLE_ROWS[version] if is_oracle else 0), c, 3, padding=1, bias=False)
        if version == 1:
            self.stem_bn = nn.BatchNorm1d(c, momentum=0.01, eps=eps)
            self.blocks = nn.Sequential(*[PostActBlock(c, eps) for _ in range(num_blocks)])
            self.act = nn.ReLU(inplace=True)
        else:
            self.blocks = nn.Sequential(*[PreActBlock(c, eps) for _ in range(num_blocks)])
            self.bn = nn.BatchNorm1d(c, momentum=0.01, eps=eps)
            self.act = nn.Mish(inplace=True)
        self.neck = nn.Conv1d(c, 32, 3, padding=1)
        self.fc = nn.Linear(32 * 34, 1024)
        if version == 1:
            self.latent = nn.Linear(1024, 512)
            self.mu_head = nn.Linear(512, 512)
            self.logsig_head = nn.Linear(512, 512)

    def forward(self, obs, invisible_obs=None):
        """phi [B, 1024] for versions 2-4, (mu, logsig) [B, 512] each for version 1, as mortal/model.py Brain.forward"""
        if self.is_oracle:
            assert invisible_obs is not None, "an oracle brain needs invisible_obs"
            obs = torch.cat((obs, invisible_obs), dim=1)
        if self.version == 1:
            x = self.blocks(self.act(self.stem_bn(self.stem(obs))))
            latent = self.act(self.latent(self.fc(self.act(self.neck(x)).flatten(1))))
            return self.mu_head(latent), self.logsig_head(latent)
        x = self.blocks(self.stem(obs))
        x = self.act(self.neck(self.act(self.bn(x))))
        return self.act(self.fc(x.flatten(1)))

    @torch.no_grad()
    def prepare_fast(self, dtype=None):
        """Inference-only fast path: eval-mode BatchNorms pre-folded into per-channel affines (two elementwise
        kernels instead of cuDNN's NCHW batch-norm kernel) and optional reduced-precision weights so that no
        autocast casts are needed. Mathematically the same network; call after loading weights / .eval()."""
        assert not self.training, "prepare_fast() is for eval mode"
        # fp32 copies of the folded affines for the fused kernels, taken before any down-cast of the parameters
        flat = lambda a: (a[0].float().flatten().contiguous(), a[1].float().flatten().contiguous())
        trunk_bn = self.stem_bn if self.version == 1 else self.bn  # the BN outside the blocks: after the stem (v1) or before the neck
        self._aff32 = [(flat(PreActBlock._affine(b.bn1)), flat(PreActBlock._affine(b.bn2))) for b in self.blocks]
        self._aff32_out = flat(PreActBlock._affine(trunk_bn))
        if dtype is not None:
            self.to(dtype)
        self._aff = [(PreActBlock._affine(b.bn1), PreActBlock._affine(b.bn2)) for b in self.blocks]
        self._aff_out = PreActBlock._affine(trunk_bn)
        # the channel-gate MLPs as fp32 copies of the (possibly down-cast) parameters, for the fused block tail
        f32 = lambda t: t.detach().float().contiguous()
        self._gate32 = [(f32(b.gate.fc1.weight), f32(b.gate.fc1.bias), f32(b.gate.fc2.weight.t()), f32(b.gate.fc2.bias)) for b in self.blocks]
        # the Conv1d kernels as (1 x 3) Conv2d kernels in channels_last, so cuDNN runs NHWC without layout round trips
        cl = lambda conv: conv.weight.unsqueeze(2).contiguous(memory_format=torch.channels_last)
        self._w = [(cl(b.conv1), cl(b.conv2)) for b in self.blocks]
        self._w_stem, self._w_neck = cl(self.stem), cl(self.neck)
        # the stem with its input channels zero-padded to a multiple of 64 (1012 -> 1024): nn_ops.obs_to_nhwc emits that layout
        cout, cin = self.stem.weight.shape[:2]
        self._cpad = (cin + 63) // 64 * 64
        wp = torch.zeros((self.stem.weight.shape[0], self._cpad, 3), dtype=self.stem.weight.dtype, device=self.stem.weight.device)
        wp[:, :cin] = self.stem.weight.detach()
        self._w_stem_pad = wp.unsqueeze(2).contiguous(memory_format=torch.channels_last)
        self._fast_dtype = dtype
        # the fused kernels take 8-channel vectors, at most 256 channels and a gate hidden layer of 1..64: other widths run unfused
        self._fusable = cout % 8 == 0 and 16 <= cout <= 256
        return self

    def forward_fast(self, obs, invisible_obs=None):
        F = torch.nn.functional
        if self.is_oracle:
            assert invisible_obs is not None, "an oracle brain needs invisible_obs"
        inv = invisible_obs if self.is_oracle else None
        fused = obs.is_cuda and self._fast_dtype == torch.bfloat16 and self._fusable
        if fused and obs.dtype == torch.float32 and obs.is_contiguous() and (
                inv is None or (inv.dtype == torch.float32 and inv.is_contiguous())):
            from . import nn_ops

            xin = nn_ops.obs_to_nhwc(obs, self._cpad) if inv is None else nn_ops.obs2_to_nhwc(obs, inv, self._cpad)
            x = F.conv2d(xin, self._w_stem_pad, padding=(0, 1))
        else:
            if inv is not None:
                obs = torch.cat((obs, inv.to(obs.dtype)), dim=1)
            if self._fast_dtype is not None:
                obs = obs.to(self._fast_dtype)
            x = obs.unsqueeze(2).contiguous(memory_format=torch.channels_last)  # [B, C, 1, 34]
            x = F.conv2d(x, self._w_stem, padding=(0, 1))
        if self.version == 1:
            return self._post_act_trunk(x, fused)
        if fused:
            # libmjx kernels (csrc/mjx_nn.cuh) around the cuDNN convolutions: per block one BN-affine+Mish pass and one pass for
            # everything between conv2 and the next block's conv1 (pooling, gate MLP, sigmoid, gate * y + x, next BN-affine+Mish)
            from . import nn_ops

            n = len(self.blocks)
            a = nn_ops.affine_mish(x, *self._aff32[0][0]) if n else nn_ops.affine_mish(x, *self._aff32_out)
            for i in range(n):
                (w1, w2), (_, (f2, g2)) = self._w[i], self._aff32[i]
                y = F.conv2d(a, w1, padding=(0, 1))
                y = F.conv2d(nn_ops.affine_mish(y, f2, g2), w2, padding=(0, 1))
                nxt = self._aff32[i + 1][0] if i + 1 < n else self._aff32_out
                x, a = nn_ops.block_tail(y, x, *self._gate32[i], *nxt)
            x = a
        else:
            for blk, aff, (w1, w2) in zip(self.blocks, self._aff, self._w):
                x = blk.forward_fast(x, aff, w1, w2, None)
            s, b = self._aff_out
            x = F.mish(torch.addcmul(b, x, s))
        x = F.mish(F.conv2d(x, self._w_neck, self.neck.bias, padding=(0, 1)))
        return F.mish(self.fc(x.flatten(1)))

    def _post_act_trunk(self, x, fused):
        """version 1 from the stem convolution's output to (mu, logsig)"""
        F = torch.nn.functional
        if fused:
            # libmjx kernels (csrc/mjx_nn.cuh): per block one BN-affine+ReLU pass, and for everything after conv2 (its BN-affine,
            # pooling, gate MLP, sigmoid, gate * t + x, ReLU) one gate kernel plus one streaming pass
            from . import nn_ops

            x = nn_ops.affine_relu(x, *self._aff32_out)
            for (w1, w2), ((f1, g1), (f2, g2)), gate in zip(self._w, self._aff32, self._gate32):
                y = F.conv2d(nn_ops.affine_relu(F.conv2d(x, w1, padding=(0, 1)), f1, g1), w2, padding=(0, 1))
                x = nn_ops.post_block_tail(y, x, f2, g2, *gate)
        else:
            s, b = self._aff_out
            x = F.relu(torch.addcmul(b, x, s))
            for blk, aff, (w1, w2) in zip(self.blocks, self._aff, self._w):
                x = blk.forward_fast(x, aff, w1, w2)
        x = F.relu(F.conv2d(x, self._w_neck, self.neck.bias, padding=(0, 1)))
        latent = F.relu(self.latent(self.fc(x.flatten(1))))
        return self.mu_head(latent), self.logsig_head(latent)


class DQN(nn.Module):
    def __init__(self, *, version: int = 4):
        super().__init__()
        if version not in OBS_ROWS:
            raise ValueError(f"unsupported Mortal version {version!r} (1..4)")
        self.version = version
        if version == 4:
            self.net = nn.Linear(1024, 1 + ACTION_SPACE)
            nn.init.zeros_(self.net.bias)
        elif version == 1:
            self.v_head = nn.Linear(512, 1)
            self.a_head = nn.Linear(512, ACTION_SPACE)
        else:
            hidden = 512 if version == 2 else 256
            self.v_head = nn.Sequential(nn.Linear(1024, hidden), nn.Mish(inplace=True), nn.Linear(hidden, 1))
            self.a_head = nn.Sequential(nn.Linear(1024, hidden), nn.Mish(inplace=True), nn.Linear(hidden, ACTION_SPACE))

    def forward(self, phi, mask):
        if self.version == 4:
            v, a = self.net(phi).split((1, ACTION_SPACE), dim=-1)
        else:
            v, a = self.v_head(phi), self.a_head(phi)
        a_mean = a.masked_fill(~mask, 0.0).sum(-1, keepdim=True) / mask.sum(-1, keepdim=True)
        return (v + a - a_mean).masked_fill(~mask, -torch.inf)


# ---- Mortal checkpoints ------------------------------------------------------------------------------------------------------

def _reference_prefixes(brain: Brain) -> dict:
    """module name in this file -> module name in mortal/model.py's Brain (an nn.Sequential `encoder.net` of the ResNet's layers)"""
    n = len(brain.blocks)
    m = {"stem": "encoder.net.0", "neck": f"encoder.net.{n + 3}", "fc": f"encoder.net.{n + 6}"}
    if brain.version == 1:  # stem, BN, ReLU, blocks, neck, ReLU, Flatten, fc
        m.update(stem_bn="encoder.net.1", latent="latent_net.0", mu_head="mu_head", logsig_head="logsig_head")
        first, unit = 3, {"conv1": 0, "bn1": 1, "conv2": 3, "bn2": 4}
    else:  # stem, blocks, BN, Mish, neck, Mish, Flatten, fc
        m["bn"] = f"encoder.net.{n + 1}"
        first, unit = 1, {"bn1": 0, "conv1": 2, "bn2": 3, "conv2": 5}
    for i in range(n):
        blk = f"encoder.net.{first + i}"
        m.update({f"blocks.{i}.{own}": f"{blk}.res_unit.{k}" for own, k in unit.items()})
        m[f"blocks.{i}.gate.fc1"], m[f"blocks.{i}.gate.fc2"] = f"{blk}.ca.shared_mlp.0", f"{blk}.ca.shared_mlp.2"
    return m


def _load_strict(module: nn.Module, given: dict, rename, what: str):
    """load `given` (reference key -> tensor) into `module`, whose key k is stored as rename(k): every key present with its
    shape and nothing else; BatchNorm's num_batches_tracked is accepted and ignored"""
    own = module.state_dict()
    want = {rename(k): k for k in own}
    out = {}
    for rk, k in want.items():
        if k.endswith(".num_batches_tracked"):
            out[k] = own[k]
            continue
        if rk not in given:
            raise KeyError(f"{what}: missing key {rk!r}")
        t = given[rk]
        if tuple(t.shape) != tuple(own[k].shape):
            raise ValueError(f"{what}: key {rk!r} has shape {tuple(t.shape)}, expected {tuple(own[k].shape)}")
        out[k] = t
    extra = [k for k in given if k not in want]
    if extra:
        raise KeyError(f"{what}: unexpected key {extra[0]!r}")
    module.load_state_dict(out)


def load_mortal(state: dict):
    """(Brain, DQN) in eval mode from a Mortal checkpoint as `torch.load` returns it (mortal/train.py:298-310:
    {'mortal': Brain.state_dict(), 'current_dqn': DQN.state_dict(), 'config': ...}). The version is the config's
    control.version (1 when absent, as mortal/player.py reads it), the width and depth its resnet section, checked against the
    tensors; an oracle brain is recognised by its stem's input width. Any missing, unexpected or misshapen key raises."""
    cfg = state["config"]
    version = cfg["control"].get("version", 1)
    if version not in OBS_ROWS:
        raise ValueError(f"unsupported Mortal version {version!r} (1..4)")
    c, n = int(cfg["resnet"]["conv_channels"]), int(cfg["resnet"]["num_blocks"])
    sd = state["mortal"]
    if "encoder.net.0.weight" not in sd:
        raise KeyError("mortal: missing key 'encoder.net.0.weight'")
    cout, cin = sd["encoder.net.0.weight"].shape[:2]
    if cout != c:
        raise ValueError(f"mortal: key 'encoder.net.0.weight' has {cout} output channels, config resnet.conv_channels is {c}")
    if cin not in (OBS_ROWS[version], OBS_ROWS[version] + ORACLE_ROWS[version]):
        raise ValueError(f"mortal: key 'encoder.net.0.weight' reads {cin} channels, which is neither the version-{version} observation "
                         f"({OBS_ROWS[version]}) nor observation + oracle rows ({OBS_ROWS[version] + ORACLE_ROWS[version]})")
    blocks = len({m.group(1) for m in map(re.compile(r"encoder\.net\.(\d+)\.(?:ca|res_unit)\.").match, sd) if m})
    if blocks != n:
        raise ValueError(f"mortal: {blocks} residual blocks in the state dict, config resnet.num_blocks is {n}")
    brain = Brain(conv_channels=c, num_blocks=n, version=version, is_oracle=cin != OBS_ROWS[version])
    names = _reference_prefixes(brain)
    _load_strict(brain, sd, lambda k: names[k.rsplit(".", 1)[0]] + "." + k.rsplit(".", 1)[1], "mortal")
    dqn = DQN(version=version)
    _load_strict(dqn, state["current_dqn"], lambda k: k, "current_dqn")
    return brain.eval(), dqn.eval()
