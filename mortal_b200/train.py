"""mortal/train.py's trainer on the device: `python -m mortal_b200.train [CONFIG]`, or `train(config, steps=None)` offline and
`train_online(config, rounds=None, steps=None)` online (`main()` runs the one `control.online` selects).

The loop of the reference's train(): batches from the device `FileDatasetsIter` (rewards from the `[grp]` GRP, as
mortal/dataloader.py:41-43 loads it), the Brain's training forward as fused kernels around cuDNN convolutions
(`Brain.forward_train`, mortal_b200.train_ops), the DQN and AuxNet heads in cuBLAS, and the dueling combine with the DQN, CQL and
next-rank losses as one kernel (`train_ops.dqn_losses`). The step is the reference's: loss = dqn + cql * min_q_weight +
next_rank * next_rank_weight, scaled by 1 / opt_step_every, GradScaler (active with enable_amp, as torch.autocast's float16),
unscale_ + clip_grad_norm_ when max_grad_norm > 0, AdamW(lr=1) under LinearWarmUpCosineAnnealingLR stepped every step.

It reads the reference's whole config.toml (the file named on the command line, else $MORTAL_CFG, else ./config.toml) and keeps
the reference's state file: `mortal` in mortal/model.py's key layout, `current_dqn`, `aux_net`, `optimizer` (its parameter groups
ordered by the reference's sorted parameter names, so the optimizer state lines up index for index), `scheduler`, `scaler`,
`steps`, `timestamp`, `best_perf`, `config`. State files move between the two trainers both ways.

Online training without `[online] actor_devices` replaces the reference's parameter server and self-play clients with one
sequential loop in one process, the reference's `force_sequential = true`. Each round plays `player.TrainPlayer.train_play_games`
sessions with the current parameters until at least `[online.server] capacity` games are held, logging each session's rankings
and the `[online] history_window` moving average as mortal/client.py does. It then runs one `selfplay.SelfPlayDatasetsIter` over
those games (the trainee's seats, the `[dataset]` flags), which yields what FileDatasetsIter yields over their written logs, so no
log is written. The step uses the online loss, dqn + next_rank * next_rank_weight with no CQL term (mortal/train.py:236-238), and saves and test-plays as offline.
Resuming from a state saved offline loads the weights, scaler, best_perf and steps, and starts a fresh optimizer and scheduler
(mortal/train.py:106-118). In this loop these keys are read and have no effect: `submit_every` (no client plays during
training) and `force_sequential` (the loop is sequential).

With `[online] actor_devices = ["cuda:1", ...]` (one self-play actor process per entry, the trainer's own device allowed),
`train_online` runs the reference's topology instead (mortal_b200.online): the actors play mortal/client.py's loop beside the
trainer, which holds mortal/server.py's state, publishes its parameters where mortal/train.py submits them (idle at start, every
`submit_every` steps, at a save off a submit, idle after each pass) and trains one pass per drain; `force_sequential` and
`capacity` act as in the reference's server. Games and parameters stay on the GPUs (CUDA IPC).

In both modes `[online.remote]`, `buffer_dir` and `drain_dir` (no files or sockets) and `[online] enable_compile` are read and
have no effect. The reference exits after a test play and respawns the trainer, a workaround for a hang in its process model;
these loops simply continue.

Data-parallel training: `torchrun --nproc-per-node=N -m mortal_b200.train [CONFIG]` starts one rank per GPU (NCCL, each rank on
cuda:LOCAL_RANK for the trainer and `[baseline.test]`), and `train()` itself trains data-parallel whenever torch.distributed is
initialised with more than one rank (NCCL or gloo). `[control] batch_size` stays the global batch: each of the W ranks trains on
batch_size / W samples, and one step is still one optimizer update over batch_size samples.
- Every training-mode BatchNorm normalises with the global batch's statistics (train_ops.bn_mish with the default group), so W
  ranks train the model one GPU would at the same batch, up to rounding. Gradients are all-reduced and averaged once per optimizer
  step, before unscale_ / clip_grad_norm_ / GradScaler.step; rank 0's initial or loaded weights are broadcast at the start, and
  from then on parameters, BatchNorm statistics, optimizer and scaler state stay bitwise equal across the ranks.
- Rank 0 builds or loads the file index, shuffles the list and broadcasts the permutation; rank r trains on the r-th contiguous
  shard of ceil(len / W) files (the reference's worker_init_fn split) with its own FileDatasetsIter. An empty shard raises
  ValueError on every rank. The ranks agree before each step (a host-side gloo collective) that every one holds a full batch;
  training ends for all when one runs out.
- The illegal-action check is all-reduced, so every rank raises the same ValueError. The loss line averages over the ranks. Only
  rank 0 logs at INFO, writes `state_file` and copies `best_state_file`; the state file is the single-process one.
- The test play splits its seeds into contiguous blocks, one per rank, each played on the rank's GPU into the same `log_dir`
  (emptied by rank 0) under the file names a single-process run uses; the ranks' Stat counters are summed, so every rank takes
  the same best_perf decision.
- Refused with ValueError: a batch_size W does not divide, a `[baseline.test]` device other than the trainer's, and
  `train_online` (online training is not data-parallel).

Differences from the reference, stated rather than hidden:
- `train()` raises ValueError for `online = true`: the online loop is `train_online`.
- Version 1 raises ValueError: its Brain returns (mu, logsig), which the reference's train.py cannot train either.
- Oracle brains are not supported: train.py never passes invisible_obs.
- `enable_compile` is read and not applied; `num_workers` has no effect (the sample stream is the in-process one, as in
  mortal_b200.train_grp, so it is not the stream of a multi-worker DataLoader for a given seed).
- There is no TensorBoard. Each save writes one `logging` line with the mean losses, the lr and the mean q / q_target; a test
  play logs its rates. Loss statistics stay on the device between saves (no host sync per step); an action outside its mask (the
  reference's assert) raises ValueError naming the step at the next save or when the call returns, whichever comes first.
"""
from __future__ import annotations

import gzip
import json
import logging
import os
import shutil
import sys
from datetime import datetime
from glob import glob
from itertools import chain
from os import path

import torch
import numpy as np
from torch import nn, optim
from torch.amp import GradScaler
from torch.nn.utils import clip_grad_norm_

from . import train_ops
from .dataloader import FileDatasetsIter
from .lr_scheduler import LinearWarmUpCosineAnnealingLR
from .model import DQN, GRP, AuxNet, Brain, _reference_key, _reference_prefixes, load_mortal_state, mortal_state_dict
from .train_grp import load_config

BEST_PERF = {"avg_rank": 4.0, "avg_pt": -135.0}


def check_config(config, world: int = 1):
    """ValueError for what the offline trainer does not run (module docstring) with `world` data-parallel ranks, before anything
    touches the device"""
    if config["control"].get("online", False):
        raise ValueError("online = true: online training runs in train_online(config), not train()")
    _check_common(config)
    if world > 1:
        batch_size = config["control"]["batch_size"]
        if batch_size % world:
            raise ValueError(f"[control] batch_size = {batch_size} is the global batch; {world} ranks must divide it")
        trainer, test = torch.device(config["control"]["device"]), torch.device(config["baseline"]["test"]["device"])
        if trainer != test:
            raise ValueError(f"data-parallel training plays each rank's test games on its trainer's device, so [baseline.test] "
                             f"device must be [control] device; got {test} and {trainer}")


def check_online_config(config, world: int = 1):
    """ValueError for an online config train_online cannot run (with `world` ranks), before anything touches the device"""
    if world > 1:
        raise ValueError(f"online training is not data-parallel: train_online runs in one process, got {world} ranks")
    _check_common(config)
    profile = os.environ.get("TRAIN_PLAY_PROFILE", "default")
    play = config.get("train_play", {}).get(profile)
    if play is None:
        raise ValueError(f"no [train_play.{profile}] profile for the trainee's self-play (TRAIN_PLAY_PROFILE selects it)")
    if play["games"] < 4:
        raise ValueError(f"[train_play.{profile}] games must be at least 4 (one seed plays 4 games), got {play['games']}")
    capacity = config["online"]["server"]["capacity"]
    if capacity < 1:
        raise ValueError(f"[online.server] capacity must be at least 1, got {capacity}")
    actor_devices = config["online"].get("actor_devices")
    if actor_devices:
        from .online import parse_actor_devices

        n, per_session = len(parse_actor_devices(actor_devices)), play["games"] // 4 * 4
        if config["online"]["server"].get("force_sequential", False) and n * per_session < capacity:
            raise ValueError(f"force_sequential = true with {n} actor(s) x {per_session} games per session = {n * per_session} "
                             f"games per round, fewer than [online.server] capacity = {capacity}: every actor would wait for "
                             "an idle publish while the trainer waits for capacity games")


def _check_common(config):
    control = config["control"]
    version = control["version"]
    if version == 1:
        raise ValueError("version 1 cannot be trained: its Brain returns (mu, logsig), which mortal/train.py cannot train either")
    if version not in (2, 3, 4):
        raise ValueError(f"unsupported Mortal version {version!r}")
    train_ops.check_channels(config["resnet"]["conv_channels"])
    if control["save_every"] % control["opt_step_every"] or control["test_every"] % control["save_every"]:
        raise ValueError("save_every must be a multiple of opt_step_every, and test_every a multiple of save_every")


def named_param_groups(brain, dqn, aux_net):
    """(decay, no_decay) lists of (reference name, parameter), as mortal/train.py:78-93 builds them: per model (Brain, DQN, AuxNet
    in that order) the Linear / Conv1d weights decay, everything else does not, each group sorted by the reference's names"""
    decay, no_decay = [], []
    brain_names = _reference_prefixes(brain)
    for model in (brain, dqn, aux_net):
        rename = (lambda k: _reference_key(brain_names, k)) if model is brain else (lambda k: k)
        params, to_decay = {}, set()
        for mod_name, mod in model.named_modules():
            for name, param in mod.named_parameters(prefix=mod_name, recurse=False):
                ref = rename(name)
                params[ref] = param
                if isinstance(mod, (nn.Linear, nn.Conv1d)) and name.endswith("weight"):
                    to_decay.add(ref)
        decay += [(n, params[n]) for n in sorted(to_decay)]
        no_decay += [(n, params[n]) for n in sorted(params.keys() - to_decay)]
    return decay, no_decay


def make_optimizer(brain, dqn, aux_net, optim_cfg):
    decay, no_decay = named_param_groups(brain, dqn, aux_net)
    groups = [{"params": [p for _, p in decay], "weight_decay": optim_cfg["weight_decay"]}, {"params": [p for _, p in no_decay]}]
    return optim.AdamW(groups, lr=1, weight_decay=0, betas=optim_cfg["betas"], eps=optim_cfg["eps"])


def _file_list(ds, player_names_set):
    """mortal/train.py:160-178: the index file's list, else the sorted (descending) recursive globs filtered to the logs one of
    the named players took part in, saved as the index"""
    file_index = ds["file_index"]
    if path.exists(file_index):
        return torch.load(file_index, weights_only=True)["file_list"]
    logging.info("building file index...")
    file_list = []
    for pat in ds["globs"]:
        file_list.extend(glob(pat, recursive=True))
    if player_names_set:
        filtered = []
        for filename in file_list:
            with gzip.open(filename, "rt") as f:
                if not set(json.loads(next(f))["names"]).isdisjoint(player_names_set):
                    filtered.append(filename)
        file_list = filtered
    file_list.sort(reverse=True)
    torch.save({"file_list": file_list}, file_index)
    return file_list


def world_info():
    """(group, rank, world) of the initialised default torch.distributed group with more than one rank, else (None, 0, 1)"""
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return dist.group.WORLD, dist.get_rank(), dist.get_world_size()
    return None, 0, 1


def shard(file_list, rank: int, world: int):
    """the rank's contiguous block of ceil(len / world) files (the reference's worker_init_fn, mortal/dataloader.py:133-139)"""
    per = -(-len(file_list) // world)
    return file_list[rank * per:(rank + 1) * per]


def check_shards(n_files: int, world: int):
    """ValueError when a rank's shard of n_files files would be empty (every rank computes the same answer)"""
    empty = [r for r in range(world) if not shard(range(n_files), r, world)]
    if empty:
        raise ValueError(f"{n_files} files cannot give each of {world} ranks a shard: rank(s) {empty} would have none")


def _player_names(ds):
    names = set()
    for filename in ds.get("player_names_files", []):
        with open(filename) as f:  # common.filtered_trimmed_lines: stripped, blank lines dropped
            names.update(s for s in (line.strip() for line in f) if s)
    return names


class _Trainer:
    """The models, optimizer, scheduler and scaler of mortal/train.py's train(), resumed from the state file, and its per-batch
    step with the saves and test plays (online: the loss has no CQL term)."""

    def __init__(self, config, online: bool):
        control = config["control"]
        self.config, self.online = config, online
        self.group, self.rank, self.world = world_info()
        self.flag_group = None  # a gloo group for host-side flags beside an NCCL default group
        if self.world > 1:
            import torch.distributed as dist

            self.flag_group = self.group if dist.get_backend() == "gloo" else dist.new_group(backend="gloo")
        self.info = logging.info if self.rank == 0 else logging.debug
        self.version = version = control["version"]
        # the rank's share of the global batch (check_config: the ranks divide it)
        self.batch_size, self.opt_step_every = control["batch_size"] // self.world, control["opt_step_every"]
        self.save_every, self.test_every = control["save_every"], control["test_every"]
        self.submit_every = control.get("submit_every")
        self.publish = None  # with self-play actors: publish(is_idle) hands the parameters over (mortal_b200.online)
        self.test_games = config["test_play"]["games"]
        self.min_q_weight = config["cql"]["min_q_weight"]
        self.next_rank_weight = config["aux"]["next_rank_weight"]
        self.gamma = config["env"]["gamma"]
        self.max_grad_norm = config["optim"]["max_grad_norm"]
        self.enable_amp = control["enable_amp"]
        _ = control.get("enable_compile", False)  # read, not applied (module docstring)

        device = torch.device(control["device"])
        if device.type != "cuda":
            raise ValueError(f"the trainer runs on a CUDA device, got {device}")
        self.device = device = torch.device("cuda", device.index if device.index is not None else torch.cuda.current_device())
        self.cudnn_benchmark = control.get("enable_cudnn_benchmark", False)
        torch.backends.cudnn.benchmark = self.cudnn_benchmark

        self.mortal = mortal = Brain(version=version, **config["resnet"]).to(device)
        self.dqn = dqn = DQN(version=version).to(device)
        self.aux_net = aux_net = AuxNet((4,)).to(device)
        self.info(f"version: {version}")
        for name, m in (("mortal", mortal), ("dqn", dqn), ("aux", aux_net)):
            self.info(f"{name} params: {sum(p.numel() for p in m.parameters() if p.requires_grad):,}")
        mortal.freeze_bn(config["freeze_bn"]["mortal"])

        self.optimizer = make_optimizer(mortal, dqn, aux_net, config["optim"])
        self.scheduler = LinearWarmUpCosineAnnealingLR(self.optimizer, **config["optim"]["scheduler"])
        self.scaler = GradScaler(device.type, enabled=self.enable_amp)
        from .player import TestPlayer

        self.test_player = TestPlayer(config)
        self.best_perf = dict(BEST_PERF)

        self.total = 0
        self.state_file, self.best_state_file = control["state_file"], control["best_state_file"]
        if path.exists(self.state_file):
            state = torch.load(self.state_file, weights_only=True, map_location=device)
            self.info(f"loaded: {datetime.fromtimestamp(state['timestamp']).strftime('%Y-%m-%d %H:%M:%S')}")
            load_mortal_state(mortal, state["mortal"])
            dqn.load_state_dict(state["current_dqn"])
            aux_net.load_state_dict(state["aux_net"])
            if not online or state["config"]["control"].get("online", False):  # mortal/train.py:113-115
                self.optimizer.load_state_dict(state["optimizer"])
                self.scheduler.load_state_dict(state["scheduler"])
            self.scaler.load_state_dict(state["scaler"])
            self.best_perf = state["best_perf"]
            self.total = state["steps"]
        if self.world > 1:  # every rank starts from rank 0's weights and BatchNorm statistics (the rest is the same file)
            import torch.distributed as dist

            for m in (mortal, dqn, aux_net):
                for t in m.state_dict().values():
                    dist.broadcast(t, 0, group=self.group)
        self.optimizer.zero_grad(set_to_none=True)
        self.info(f"device: {device} ({torch.cuda.get_device_name(device)})"
                  + (f", rank {self.rank} of {self.world}" if self.world > 1 else ""))

        zero = lambda: torch.zeros((), dtype=torch.float64, device=device)
        self._zero = zero
        self.stats = {k: zero() for k in ("dqn_loss", "cql_loss", "next_rank_loss")}
        self.all_q = torch.zeros((self.save_every, self.batch_size), dtype=torch.float32, device=device)
        self.all_q_target = torch.zeros_like(self.all_q)
        self.bad_steps = torch.zeros(self.save_every, dtype=torch.int32, device=device)
        self.idx = 0

    def all_ranks(self, flag: bool) -> bool:
        """True when `flag` holds on every rank (a host-side collective: no device synchronisation)"""
        if self.world == 1:
            return flag
        import torch.distributed as dist

        t = torch.tensor([int(flag)], dtype=torch.int32)
        dist.all_reduce(t, op=dist.ReduceOp.MIN, group=self.flag_group)
        return bool(t.item())

    def _mean_over_ranks(self, *scalars):
        """each device scalar averaged over the ranks (as they are with one rank)"""
        if self.world == 1:
            return scalars
        import torch.distributed as dist

        t = torch.stack([s.double() for s in scalars])
        dist.all_reduce(t, group=self.group)
        return (t / self.world).unbind()

    def _all_reduce_grads(self):
        """sum the gradients over the ranks (one flat all-reduce) and divide by the rank count: the gradient of the global
        batch's mean loss, bit-identical on every rank"""
        import torch.distributed as dist

        grads = [p.grad for g in self.optimizer.param_groups for p in g["params"] if p.grad is not None]
        flat = torch.cat([g.reshape(-1) for g in grads])
        dist.all_reduce(flat, group=self.group)
        flat /= self.world
        o = 0
        for g in grads:
            g.copy_(flat[o:o + g.numel()].view_as(g))
            o += g.numel()

    def check_actions(self):
        """ValueError naming the first step since the last check whose batch had an action outside its mask (on any rank: every
        rank raises the same error)"""
        bad = self.bad_steps[:self.idx]
        if self.world > 1:
            import torch.distributed as dist

            bad = bad.clone()
            dist.all_reduce(bad, group=self.group)
        hit = torch.nonzero(bad).flatten().tolist()
        if hit:
            raise ValueError(f"step {self.total - self.idx + hit[0] + 1}: an action of the batch is not legal in its mask")

    def step(self, obs, actions, masks, steps_to_done, kyoku_rewards, player_ranks):
        """one training step on a full batch, then the save and the test play when they are due"""
        mortal, dqn, aux_net = self.mortal, self.dqn, self.aux_net
        with torch.autocast(self.device.type, enabled=self.enable_amp):
            phi = mortal.forward_train(obs, group=self.group)
            v, a = dqn.heads(phi)
            next_rank_logits, = aux_net(phi)
            dqn_loss, cql_loss, next_rank_loss, q, q_target, bad = train_ops.dqn_losses(
                v, a, next_rank_logits, masks, actions, steps_to_done, kyoku_rewards, player_ranks, self.gamma)
            if self.online:  # mortal/train.py:236-238: no CQL term (its output gets no gradient)
                loss = dqn_loss + next_rank_loss * self.next_rank_weight
            else:
                loss = dqn_loss + cql_loss * self.min_q_weight + next_rank_loss * self.next_rank_weight
        self.scaler.scale(loss / self.opt_step_every).backward()

        idx = self.idx
        with torch.no_grad():
            self.stats["dqn_loss"] += dqn_loss
            if not self.online:
                self.stats["cql_loss"] += cql_loss
            self.stats["next_rank_loss"] += next_rank_loss
            self.all_q[idx] = q
            self.all_q_target[idx] = q_target
            self.bad_steps[idx] = bad
        self.total += 1
        self.idx += 1
        if self.idx % self.opt_step_every == 0:
            if self.world > 1:
                self._all_reduce_grads()
            if self.max_grad_norm > 0:
                self.scaler.unscale_(self.optimizer)
                clip_grad_norm_(chain.from_iterable(g["params"] for g in self.optimizer.param_groups), self.max_grad_norm)
            self.scaler.step(self.optimizer)
            self.scaler.update()
            self.optimizer.zero_grad(set_to_none=True)
        self.scheduler.step()
        if self.publish is not None and self.total % self.submit_every == 0:  # mortal/train.py:271-273
            self.publish(False)
        if self.total % self.save_every == 0:
            self._save()

    def _save(self):
        total, test_every, stats = self.total, self.test_every, self.stats
        self.check_actions()
        n = self.save_every
        dqn_loss, cql_loss, next_rank_loss, q, q_target = self._mean_over_ranks(
            stats["dqn_loss"], stats["cql_loss"], stats["next_rank_loss"], self.all_q.mean(), self.all_q_target.mean())
        cql = "" if self.online else f" cql_loss {(cql_loss / n).item():.6f}"
        self.info(f"steps {total:,}: dqn_loss {(dqn_loss / n).item():.6f}{cql} "
                  f"next_rank_loss {(next_rank_loss / n).item():.6f} lr {self.scheduler.get_last_lr()[0]:.4e} "
                  f"q {q.item():.6f} q_target {q_target.item():.6f}")
        for k in stats:
            stats[k] = self._zero()
        self.idx = 0
        self.info(f"total steps: {total:,} (~{(test_every - total % test_every) % test_every:,})")
        state = None if self.rank else {
            "mortal": mortal_state_dict(self.mortal),
            "current_dqn": self.dqn.state_dict(),
            "aux_net": self.aux_net.state_dict(),
            "optimizer": self.optimizer.state_dict(),
            "scheduler": self.scheduler.state_dict(),
            "scaler": self.scaler.state_dict(),
            "steps": total,
            "timestamp": datetime.now().timestamp(),
            "best_perf": self.best_perf,
            "config": self.config,
        }
        if state is not None:
            torch.save(state, self.state_file)
        if self.publish is not None and total % self.submit_every != 0:  # mortal/train.py:312-314
            self.publish(False)

        if total % test_every == 0:
            best_perf = self.best_perf
            stat = self.test_player.test_play(self.test_games // 4, self.mortal, self.dqn, self.device, group=self.group)
            self.mortal.train()
            self.dqn.train()
            avg_pt = stat.avg_pt([90, 45, 0, -135])  # for display only, never used in training
            better = avg_pt >= best_perf["avg_pt"] and stat.avg_rank <= best_perf["avg_rank"]
            if better:
                past_best = best_perf.copy()
                best_perf["avg_pt"] = avg_pt
                best_perf["avg_rank"] = stat.avg_rank
            self.info(f"avg rank: {stat.avg_rank:.6}")
            self.info(f"avg pt: {avg_pt:.6}")
            self.info("test play: rank 1/2/3/4 {:.4f} {:.4f} {:.4f} {:.4f}; agari {:.4f} houjuu {:.4f} fuuro {:.4f} "
                         "riichi {:.4f}; point per agari {:.1f} (riichi {:.1f}, fuuro {:.1f}, dama {:.1f}), per houjuu {:.1f}, "
                         "per round {:.1f}; jun agari {:.2f} houjuu {:.2f} riichi {:.2f}; after riichi agari {:.4f} houjuu "
                         "{:.4f}, chasing {:.4f}, chased {:.4f}, riichi point {:.1f}; after fuuro agari {:.4f} houjuu {:.4f}, "
                         "fuuro num {:.4f}, fuuro point {:.1f}".format(
                             stat.rank_1_rate, stat.rank_2_rate, stat.rank_3_rate, stat.rank_4_rate, stat.agari_rate,
                             stat.houjuu_rate, stat.fuuro_rate, stat.riichi_rate, stat.avg_point_per_agari,
                             stat.avg_point_per_riichi_agari, stat.avg_point_per_fuuro_agari, stat.avg_point_per_dama_agari,
                             stat.avg_point_per_houjuu, stat.avg_point_per_round, stat.avg_agari_jun, stat.avg_houjuu_jun,
                             stat.avg_riichi_jun, stat.agari_rate_after_riichi, stat.houjuu_rate_after_riichi,
                             stat.chasing_riichi_rate, stat.riichi_chased_rate, stat.avg_riichi_point,
                             stat.agari_rate_after_fuuro, stat.houjuu_rate_after_fuuro, stat.avg_fuuro_num, stat.avg_fuuro_point))
            if better and state is not None:
                torch.save(state, self.state_file)
                logging.info(f"a new record has been made, pt: {past_best['avg_pt']:.4} -> {best_perf['avg_pt']:.4}, "
                             f"rank: {past_best['avg_rank']:.4} -> {best_perf['avg_rank']:.4}, saving to {self.best_state_file}")
                shutil.copy(self.state_file, self.best_state_file)


def _load_grp(config):
    grp = GRP(**config["grp"]["network"])
    grp.load_state_dict(torch.load(config["grp"]["state_file"], weights_only=True, map_location=torch.device("cpu"))["model"])
    return grp


def train(config, steps=None):
    """mortal/train.py train() over the whole config (dict), offline: one pass over the file list, as the reference runs. `steps`
    bounds this call to that many training steps (None: until the data ends). Returns (brain, dqn, aux_net, optimizer, total
    steps)."""
    world = world_info()[2]
    check_config(config, world)
    T = _Trainer(config, online=False)
    ds = config["dataset"]
    grp = _load_grp(config)
    player_names_set = _player_names(ds)
    T.info(f"loaded {len(player_names_set):,} players")
    file_list = shard_file_list(ds, player_names_set, T) if world > 1 else _file_list(ds, player_names_set)
    T.info(f"file list size: {len(file_list):,}")
    T.info(f"total steps: {T.total:,} (~{(T.test_every - T.total % T.test_every) % T.test_every:,})")
    file_data = FileDatasetsIter(T.version, file_list, config["env"]["pts"], file_batch_size=ds["file_batch_size"],
                                 reserve_ratio=ds["reserve_ratio"], player_names=list(player_names_set), num_epochs=ds["num_epochs"],
                                 enable_augmentation=ds["enable_augmentation"], augmented_first=ds["augmented_first"], grp=grp,
                                 batch_size=T.batch_size, device=T.device.index)
    done = 0
    if world == 1:
        for batch in file_data:
            if steps is not None and done >= steps:
                break
            if batch[0].shape[0] != T.batch_size:
                continue  # a final short batch is not trained on (mortal/train.py:389-422)
            T.step(*batch)
            done += 1
    else:
        batches = iter(file_data)
        while steps is None or done < steps:
            batch = next(batches, None)
            # every rank steps or none does: training ends for all when one rank's shard runs out (its final short batch
            # included, which is not trained on, as above)
            if not T.all_ranks(batch is not None and batch[0].shape[0] == T.batch_size):
                break
            T.step(*batch)
            done += 1
    T.check_actions()
    return T.mortal, T.dqn, T.aux_net, T.optimizer, T.total


def shard_file_list(ds, player_names_set, T):
    """this rank's shard of the file list: rank 0 builds or loads the index while the others wait, every rank loads it, rank 0
    shuffles it and broadcasts the permutation, and each rank takes its contiguous block (ValueError on every rank when a block
    would be empty)"""
    import torch.distributed as dist

    if T.rank == 0:
        _file_list(ds, player_names_set)
    dist.barrier(group=T.flag_group)
    file_list = _file_list(ds, player_names_set)
    check_shards(len(file_list), T.world)
    perm = torch.randperm(len(file_list)) if T.rank == 0 else torch.empty(len(file_list), dtype=torch.int64)
    dist.broadcast(perm, 0, group=T.flag_group)
    return shard([file_list[i] for i in perm.tolist()], T.rank, T.world)


def _train_pass(T, config, grp, games, steps, done):
    """one SelfPlayDatasetsIter pass over `games` (the trainee's seats, the [dataset] flags), stopping once `done` reaches `steps`
    -> the new `done`"""
    from .selfplay import SelfPlayDatasetsIter

    ds = config["dataset"]
    data = SelfPlayDatasetsIter(T.version, games, config["env"]["pts"], file_batch_size=ds["file_batch_size"],
                                reserve_ratio=ds["reserve_ratio"], player_names=["trainee"], num_epochs=ds["num_epochs"],
                                enable_augmentation=ds["enable_augmentation"], augmented_first=ds["augmented_first"], grp=grp,
                                batch_size=T.batch_size, device=T.device.index)
    for batch in data:
        if steps is not None and done >= steps:
            break
        if batch[0].shape[0] != T.batch_size:
            continue  # a final short batch is not trained on (mortal/train.py:389-422)
        T.step(*batch)
        done += 1
    return done


def train_online(config, rounds=None, steps=None, monitor=None):
    """mortal/train.py with `online = true` (module docstring). Without `[online] actor_devices`, one sequential loop in this
    process: `rounds` bounds the call to that many rounds of self-play + training. With it, self-play actors beside the trainer
    (mortal_b200.online.train_concurrent): `rounds` counts the drains trained on, and `monitor(kind, **info)` receives the
    parameter server's publish, submit and drain events (mortal_b200.online.Server). `steps` bounds either to that many training
    steps (None: no bound; the loop then runs until interrupted). Returns (brain, dqn, aux_net, optimizer, total steps)."""
    from .player import TrainPlayer
    from .selfplay import SelfPlayGames

    check_online_config(config, world_info()[2])
    if config["online"].get("actor_devices"):
        from .online import train_concurrent

        return train_concurrent(config, rounds=rounds, steps=steps, monitor=monitor)
    online_cfg = config["online"]
    server = online_cfg["server"]
    capacity, history_window = server["capacity"], online_cfg["history_window"]
    _ = (config["control"].get("submit_every"), server.get("force_sequential"), server.get("buffer_dir"),  # read, no effect
         server.get("drain_dir"), online_cfg.get("remote"), online_cfg.get("enable_compile"))       # (module docstring)
    T = _Trainer(config, online=True)
    grp = _load_grp(config)
    train_player = TrainPlayer(config)
    pts = np.array([90, 45, 0, -135])  # mortal/client.py:31, for the log lines only
    history = []
    done = rounds_done = 0
    while (rounds is None or rounds_done < rounds) and (steps is None or done < steps):
        held, n_games = [], 0
        while n_games < capacity:  # mortal/client.py:54-65, one session at a time
            rankings, games = train_player.train_play_games(T.mortal, T.dqn, T.device)
            held.append(games)
            n_games += len(games)
            history.append(np.array(rankings))
            if len(history) > history_window:
                del history[0]
            total_r = np.sum(history, axis=0)
            logging.info(f"trainee rankings: {rankings} ({rankings @ np.arange(1, 5) / rankings.sum():.6}, "
                         f"{rankings @ pts / rankings.sum():.6}pt)")
            logging.info(f"last {len(history)} sessions: {total_r} ({total_r @ np.arange(1, 5) / total_r.sum():.6}, "
                         f"{total_r @ pts / total_r.sum():.6}pt)")
        games = SelfPlayGames.concat(held)
        del held
        logging.info(f"round {rounds_done + 1}: {len(games):,} games; total steps: {T.total:,} "
                     f"(~{(T.test_every - T.total % T.test_every) % T.test_every:,})")
        done = _train_pass(T, config, grp, games, steps, done)
        del games  # the round's games are freed before the next round plays
        rounds_done += 1
    T.check_actions()
    return T.mortal, T.dqn, T.aux_net, T.optimizer, T.total


def main(argv=None):
    """`python -m mortal_b200.train [CONFIG]`; under torchrun (WORLD_SIZE > 1) one data-parallel rank on cuda:LOCAL_RANK over NCCL"""
    argv = sys.argv[1:] if argv is None else argv
    logging.basicConfig(level=logging.INFO, format="%(asctime)s %(levelname)s %(message)s")
    distributed = int(os.environ.get("WORLD_SIZE", "1")) > 1
    try:
        config = load_config(argv[0] if argv else None)
        if distributed:
            import torch.distributed as dist

            device = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
            torch.cuda.set_device(device)
            dist.init_process_group("nccl", device_id=device)
            config["control"]["device"] = config["baseline"]["test"]["device"] = str(device)
        (train_online if config["control"].get("online", False) else train)(config)
    except KeyboardInterrupt:
        pass
    finally:
        if distributed:
            import torch.distributed as dist

            if dist.is_initialized():
                dist.destroy_process_group()


if __name__ == "__main__":
    main()
