"""mortal/train.py's offline trainer on the device: `python -m mortal_b200.train [CONFIG]`, or `train(config, steps=None)`.

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

Differences from the reference, stated rather than hidden:
- `online = true` raises ValueError: online training needs the reference's parameter server and self-play clients (submit_param,
  drain, TrainPlayer), which are not built.
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
import shutil
import sys
from datetime import datetime
from glob import glob
from itertools import chain
from os import path

import torch
from torch import nn, optim
from torch.amp import GradScaler
from torch.nn.utils import clip_grad_norm_

from . import train_ops
from .dataloader import FileDatasetsIter
from .lr_scheduler import LinearWarmUpCosineAnnealingLR
from .model import DQN, GRP, AuxNet, Brain, _reference_key, _reference_prefixes, load_mortal_state, mortal_state_dict
from .train_grp import load_config

BEST_PERF = {"avg_rank": 4.0, "avg_pt": -135.0}


def check_config(config):
    """ValueError for what this trainer does not build (module docstring), before anything touches the device"""
    control = config["control"]
    if control.get("online", False):
        raise ValueError("online training is not supported: it needs the reference's parameter server and self-play clients "
                         "(submit_param, drain, TrainPlayer)")
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


def _player_names(ds):
    names = set()
    for filename in ds.get("player_names_files", []):
        with open(filename) as f:  # common.filtered_trimmed_lines: stripped, blank lines dropped
            names.update(s for s in (line.strip() for line in f) if s)
    return names


def train(config, steps=None):
    """mortal/train.py train() over the whole config (dict), offline: one pass over the file list, as the reference runs. `steps`
    bounds this call to that many training steps (None: until the data ends). Returns (brain, dqn, aux_net, optimizer, total
    steps)."""
    check_config(config)
    control = config["control"]
    version = control["version"]
    batch_size, opt_step_every = control["batch_size"], control["opt_step_every"]
    save_every, test_every = control["save_every"], control["test_every"]
    test_games = config["test_play"]["games"]
    min_q_weight = config["cql"]["min_q_weight"]
    next_rank_weight = config["aux"]["next_rank_weight"]
    gamma, pts = config["env"]["gamma"], config["env"]["pts"]
    ds = config["dataset"]
    optim_cfg = config["optim"]
    max_grad_norm = optim_cfg["max_grad_norm"]
    enable_amp = control["enable_amp"]
    _ = control.get("enable_compile", False)  # read, not applied (module docstring)

    device = torch.device(control["device"])
    if device.type != "cuda":
        raise ValueError(f"the trainer runs on a CUDA device, got {device}")
    device = torch.device("cuda", device.index if device.index is not None else torch.cuda.current_device())
    torch.backends.cudnn.benchmark = control.get("enable_cudnn_benchmark", False)

    mortal = Brain(version=version, **config["resnet"]).to(device)
    dqn = DQN(version=version).to(device)
    aux_net = AuxNet((4,)).to(device)
    logging.info(f"version: {version}")
    for name, m in (("mortal", mortal), ("dqn", dqn), ("aux", aux_net)):
        logging.info(f"{name} params: {sum(p.numel() for p in m.parameters() if p.requires_grad):,}")
    mortal.freeze_bn(config["freeze_bn"]["mortal"])

    optimizer = make_optimizer(mortal, dqn, aux_net, optim_cfg)
    scheduler = LinearWarmUpCosineAnnealingLR(optimizer, **optim_cfg["scheduler"])
    scaler = GradScaler(device.type, enabled=enable_amp)
    from .player import TestPlayer

    test_player = TestPlayer(config)
    best_perf = dict(BEST_PERF)

    total = 0
    state_file, best_state_file = control["state_file"], control["best_state_file"]
    if path.exists(state_file):
        state = torch.load(state_file, weights_only=True, map_location=device)
        logging.info(f"loaded: {datetime.fromtimestamp(state['timestamp']).strftime('%Y-%m-%d %H:%M:%S')}")
        load_mortal_state(mortal, state["mortal"])
        dqn.load_state_dict(state["current_dqn"])
        aux_net.load_state_dict(state["aux_net"])
        optimizer.load_state_dict(state["optimizer"])
        scheduler.load_state_dict(state["scheduler"])
        scaler.load_state_dict(state["scaler"])
        best_perf = state["best_perf"]
        total = state["steps"]
    optimizer.zero_grad(set_to_none=True)
    logging.info(f"device: {device} ({torch.cuda.get_device_name(device)})")

    grp = GRP(**config["grp"]["network"])
    grp.load_state_dict(torch.load(config["grp"]["state_file"], weights_only=True, map_location=torch.device("cpu"))["model"])
    player_names_set = _player_names(ds)
    logging.info(f"loaded {len(player_names_set):,} players")
    file_list = _file_list(ds, player_names_set)
    logging.info(f"file list size: {len(file_list):,}")
    logging.info(f"total steps: {total:,} (~{(test_every - total % test_every) % test_every:,})")
    file_data = FileDatasetsIter(version, file_list, pts, file_batch_size=ds["file_batch_size"], reserve_ratio=ds["reserve_ratio"],
                                 player_names=list(player_names_set), num_epochs=ds["num_epochs"],
                                 enable_augmentation=ds["enable_augmentation"], augmented_first=ds["augmented_first"], grp=grp,
                                 batch_size=batch_size, device=device.index)

    zero = lambda: torch.zeros((), dtype=torch.float64, device=device)
    stats = {k: zero() for k in ("dqn_loss", "cql_loss", "next_rank_loss")}
    all_q = torch.zeros((save_every, batch_size), dtype=torch.float32, device=device)
    all_q_target = torch.zeros_like(all_q)
    bad_steps = torch.zeros(save_every, dtype=torch.int32, device=device)
    idx = 0

    def check_actions(first_step):
        """ValueError naming the first step since the last check whose batch had an action outside its mask"""
        hit = torch.nonzero(bad_steps[:idx]).flatten().tolist()
        if hit:
            raise ValueError(f"step {first_step + hit[0] + 1}: an action of the batch is not legal in its mask")

    done = 0
    for obs, actions, masks, steps_to_done, kyoku_rewards, player_ranks in file_data:
        if steps is not None and done >= steps:
            break
        if obs.shape[0] != batch_size:
            continue  # a final short batch is not trained on (mortal/train.py:389-422)
        with torch.autocast(device.type, enabled=enable_amp):
            phi = mortal.forward_train(obs)
            v, a = dqn.heads(phi)
            next_rank_logits, = aux_net(phi)
            dqn_loss, cql_loss, next_rank_loss, q, q_target, bad = train_ops.dqn_losses(
                v, a, next_rank_logits, masks, actions, steps_to_done, kyoku_rewards, player_ranks, gamma)
            loss = dqn_loss + cql_loss * min_q_weight + next_rank_loss * next_rank_weight
        scaler.scale(loss / opt_step_every).backward()

        with torch.no_grad():
            stats["dqn_loss"] += dqn_loss
            stats["cql_loss"] += cql_loss
            stats["next_rank_loss"] += next_rank_loss
            all_q[idx] = q
            all_q_target[idx] = q_target
            bad_steps[idx] = bad
        total += 1
        done += 1
        idx += 1
        if idx % opt_step_every == 0:
            if max_grad_norm > 0:
                scaler.unscale_(optimizer)
                clip_grad_norm_(chain.from_iterable(g["params"] for g in optimizer.param_groups), max_grad_norm)
            scaler.step(optimizer)
            scaler.update()
            optimizer.zero_grad(set_to_none=True)
        scheduler.step()

        if total % save_every == 0:
            check_actions(total - idx)
            n = save_every
            logging.info(f"steps {total:,}: dqn_loss {(stats['dqn_loss'] / n).item():.6f} cql_loss {(stats['cql_loss'] / n).item():.6f} "
                         f"next_rank_loss {(stats['next_rank_loss'] / n).item():.6f} lr {scheduler.get_last_lr()[0]:.4e} "
                         f"q {all_q.mean().item():.6f} q_target {all_q_target.mean().item():.6f}")
            for k in stats:
                stats[k] = zero()
            idx = 0
            logging.info(f"total steps: {total:,} (~{(test_every - total % test_every) % test_every:,})")
            state = {
                "mortal": mortal_state_dict(mortal),
                "current_dqn": dqn.state_dict(),
                "aux_net": aux_net.state_dict(),
                "optimizer": optimizer.state_dict(),
                "scheduler": scheduler.state_dict(),
                "scaler": scaler.state_dict(),
                "steps": total,
                "timestamp": datetime.now().timestamp(),
                "best_perf": best_perf,
                "config": config,
            }
            torch.save(state, state_file)

            if total % test_every == 0:
                stat = test_player.test_play(test_games // 4, mortal, dqn, device)
                mortal.train()
                dqn.train()
                avg_pt = stat.avg_pt([90, 45, 0, -135])  # for display only, never used in training
                better = avg_pt >= best_perf["avg_pt"] and stat.avg_rank <= best_perf["avg_rank"]
                if better:
                    past_best = best_perf.copy()
                    best_perf["avg_pt"] = avg_pt
                    best_perf["avg_rank"] = stat.avg_rank
                logging.info(f"avg rank: {stat.avg_rank:.6}")
                logging.info(f"avg pt: {avg_pt:.6}")
                logging.info("test play: rank 1/2/3/4 {:.4f} {:.4f} {:.4f} {:.4f}; agari {:.4f} houjuu {:.4f} fuuro {:.4f} "
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
                if better:
                    torch.save(state, state_file)
                    logging.info(f"a new record has been made, pt: {past_best['avg_pt']:.4} -> {best_perf['avg_pt']:.4}, "
                                 f"rank: {past_best['avg_rank']:.4} -> {best_perf['avg_rank']:.4}, saving to {best_state_file}")
                    shutil.copy(state_file, best_state_file)
    check_actions(total - idx)
    return mortal, dqn, aux_net, optimizer, total


def main(argv=None):
    argv = sys.argv[1:] if argv is None else argv
    logging.basicConfig(level=logging.INFO, format="%(asctime)s %(levelname)s %(message)s")
    try:
        train(load_config(argv[0] if argv else None))
    except KeyboardInterrupt:
        pass


if __name__ == "__main__":
    main()
