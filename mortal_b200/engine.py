"""Engines: the decision makers the environment calls back into.

`DeviceEngine` is the zero-copy fast path: it consumes the on-device observation / mask tensors and returns
on-device actions, with the selection semantics of mortal/engine.py:43-94 (masked dueling Q, greedy argmax or
epsilon-Boltzmann with top-p). Any object following the reference's duck-typed protocol
(agent/mortal.rs:54-74, 126-152: `engine_type == 'mortal'`, `react_batch(list[np], list[np], None)`)
still works through `HostProtocolEngine`, which pays the device->host->device round trip the reference pays.
"""
from __future__ import annotations

import copy

import numpy as np
import torch


class DeviceEngine:
    engine_type = "mortal"

    def __init__(self, brain, dqn, *, version=4, device=None, enable_amp=True, enable_quick_eval=True,
                 enable_rule_based_agari_guard=False, name="NoName", boltzmann_epsilon=0.0, boltzmann_temp=1.0,
                 top_p=1.0, is_oracle=False, stochastic_latent=False, fast_inference=True):
        self.device = device or torch.device("cuda")
        self.brain = brain.to(self.device).eval()
        self.dqn = dqn.to(self.device).eval()
        # BN-folded bf16 inference path when the brain offers one (mortal_b200.model.Brain); plain autocast otherwise
        self.fast = bool(fast_inference and enable_amp and hasattr(self.brain, "prepare_fast") and self.device.type == "cuda")
        self._fast_brain = None
        if self.fast:
            from . import _lib

            _lib.init(self.device.index or 0)  # the fused elementwise kernels live in libmjx
            self.refresh()
        self.version = version
        self.is_oracle = is_oracle
        self.enable_amp = enable_amp
        self.enable_quick_eval = enable_quick_eval
        self.enable_rule_based_agari_guard = enable_rule_based_agari_guard
        self.name = name
        self.boltzmann_epsilon = boltzmann_epsilon
        self.boltzmann_temp = boltzmann_temp
        self.top_p = top_p
        self.stochastic_latent = stochastic_latent  # version 1: sample the latent from Normal(mu, exp(logsig) + 1e-6) instead of mu
        self._graphs = {}

    @torch.no_grad()
    def refresh(self):
        """(Re)build the bf16 BN-folded inference copy from the caller's module. The caller's `brain` is never touched:
        mortal/train.py:317 and player.py:120 hand the live training model to the engine and keep training it afterwards, so its
        fp32 parameters and BatchNorm statistics must survive. Call again after the weights changed."""
        if self.fast:
            self._fast_brain = copy.deepcopy(self.brain).eval()
            self._fast_brain.prepare_fast(torch.bfloat16)
            self._graphs = {}

    @torch.inference_mode()
    def react_device(self, obs: torch.Tensor, masks: torch.Tensor, return_greedy: bool = False, invisible_obs=None):
        """obs [B, C, 34] f32 cuda, masks [B, 46] bool cuda (invisible_obs [B, 211 | 217, 34] f32 cuda for oracle engines)
        -> (actions int64 [B], q [B, 46][, is_greedy bool [B]])"""
        inv = (invisible_obs,) if self.is_oracle else ()
        if self.fast:
            q = self.dqn(self._latent(self._fast_brain.forward_fast(obs, *inv)).float(), masks)
        else:
            with torch.autocast(self.device.type, dtype=torch.bfloat16, enabled=self.enable_amp):
                q = self.dqn(self._latent(self.brain(obs, *inv)), masks)
        if self.boltzmann_epsilon > 0:
            b = obs.shape[0]
            greedy = torch.full((b,), 1 - self.boltzmann_epsilon, device=self.device).bernoulli().to(torch.bool)
            logits = (q / self.boltzmann_temp).masked_fill(~masks, -torch.inf)
            sampled = sample_top_p(logits, self.top_p)
            actions = torch.where(greedy, q.argmax(-1), sampled)
        else:
            actions = q.argmax(-1)
            greedy = None
        if return_greedy:
            if greedy is None:
                greedy = torch.ones(obs.shape[0], dtype=torch.bool, device=self.device)
            return actions, q, greedy
        return actions, q

    def _latent(self, out):
        """version 1 brains return (mu, logsig) (mortal/engine.py:60-66): the DQN gets mu, or a sample with stochastic_latent"""
        if not isinstance(out, tuple):
            return out
        mu, logsig = out
        if self.stochastic_latent:
            return torch.distributions.Normal(mu, logsig.exp() + 1e-6).sample()
        return mu

    @torch.inference_mode()
    def react_static(self, obs_buf: torch.Tensor, masks_buf: torch.Tensor, nr: int, bucket: int = 256):
        """react_device(obs_buf[:nr], masks_buf[:nr]) for PERSISTENT buffers (BatchEnv.obs_buffer() / .masks): the forward
        over the first ceil(nr / bucket) * bucket rows is captured once per bucket as a CUDA graph and replayed, which
        removes the ~600 kernel-launch calls per step from the host. Greedy, non-oracle engines with a deterministic latent
        only; rows past nr are stale and ignored."""
        if self.boltzmann_epsilon > 0 or not self.fast or self.is_oracle or self.stochastic_latent:
            return self.react_device(obs_buf[:nr], masks_buf[:nr])
        nb = min(((nr + bucket - 1) // bucket) * bucket, obs_buf.shape[0])
        key = (obs_buf.data_ptr(), masks_buf.data_ptr(), nb)
        entry = self._graphs.get(key)
        if entry is None:
            cur = torch.cuda.current_stream(self.device)
            side = torch.cuda.Stream(self.device)
            side.wait_stream(cur)
            with torch.cuda.stream(side):  # warm-up outside the capture (cuDNN algorithm selection, lazy init)
                for _ in range(2):
                    self.react_device(obs_buf[:nb], masks_buf[:nb])
            cur.wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                a, q = self.react_device(obs_buf[:nb], masks_buf[:nb])
            entry = (graph, a, q)
            self._graphs[key] = entry
        entry[0].replay()
        return entry[1][:nr], entry[2][:nr]

    # the reference protocol, for callers that only know libriichi's calling convention
    def react_batch(self, obs, masks, invisible_obs):
        o = torch.as_tensor(_stack_rows(obs), device=self.device)
        m = torch.as_tensor(_stack_rows(masks), device=self.device)
        inv = None if invisible_obs is None else torch.as_tensor(_stack_rows(invisible_obs), device=self.device)
        actions, q, greedy = self.react_device(o, m, return_greedy=True, invisible_obs=inv)
        return actions.tolist(), q.float().tolist(), m.tolist(), greedy.tolist()


def _stack_rows(rows):
    """np.stack(rows) without the copy when the rows already are consecutive slices of one buffer — which is how the arena hands
    them out (views over the pinned buffer mjx_env_encode_obs_host filled), so the H2D copy then reads pinned memory directly."""
    first = rows[0]
    n, step = len(rows), first.nbytes
    if n > 1 and first.flags.c_contiguous and step:
        p0 = first.__array_interface__["data"][0]
        if all(r.__array_interface__["data"][0] == p0 + i * step and r.shape == first.shape and r.dtype == first.dtype
               for i, r in enumerate(rows)):
            return np.lib.stride_tricks.as_strided(first, shape=(n, *first.shape), strides=(step, *first.strides), writeable=bool(first.flags.writeable))
    return np.stack(rows, axis=0)


def sample_top_p(logits, p):
    """Nucleus sampling over the last axis: draw from the smallest set of highest-probability actions whose mass reaches
    `p` (engine.py:83-94 semantics: p >= 1 is plain categorical sampling, p <= 0 the argmax)."""
    if p >= 1:
        return torch.distributions.Categorical(logits=logits).sample()
    if p <= 0:
        return logits.argmax(-1)
    order = logits.argsort(-1, descending=True)
    mass = logits.gather(-1, order).softmax(-1)
    before = mass.cumsum(-1) - mass               # probability mass ranked strictly above each action
    nucleus = torch.where(before <= p, mass, torch.zeros_like(mass))
    pick = nucleus.multinomial(1)                 # multinomial renormalises the kept mass itself
    return order.gather(-1, pick).squeeze(-1)


class HostProtocolEngine:
    """Adapter: drives a reference-style engine (react_batch over lists of numpy arrays) from device rows."""

    def __init__(self, engine):
        assert getattr(engine, "engine_type", None) == "mortal", "only engine_type='mortal' is supported"
        self.engine = engine
        for attr in ("name", "version", "is_oracle", "enable_quick_eval", "enable_rule_based_agari_guard"):
            setattr(self, attr, getattr(engine, attr))

    def react_host(self, obs_np: np.ndarray, masks_np: np.ndarray, idx: np.ndarray, inv_np=None):
        """rows `idx` of host arrays (views over pinned buffers filled by mjx_env_encode_obs_host) -> (actions, q, is_greedy) numpy,
        through the reference protocol: lists of per-row arrays in, lists out (agent/mortal.rs:126-152)."""
        invisible = None if inv_np is None else [inv_np[i] for i in idx]  # mortal.rs:137-146: Some(list) for oracle engines only
        actions, q, _, greedy = self.engine.react_batch([obs_np[i] for i in idx], [masks_np[i] for i in idx], invisible)
        return np.asarray(actions, dtype=np.int64), np.asarray(q, dtype=np.float32), np.asarray(greedy, dtype=bool)

    def react_device(self, obs: torch.Tensor, masks: torch.Tensor, invisible_obs=None):
        obs_h = obs.cpu().numpy()
        masks_h = masks.cpu().numpy()
        inv = None if invisible_obs is None else list(invisible_obs.cpu().numpy())
        actions, q, _, _ = self.engine.react_batch(list(obs_h), list(masks_h), inv)
        dev = obs.device
        return torch.as_tensor(actions, dtype=torch.int64, device=dev), torch.as_tensor(q, dtype=torch.float32, device=dev)
