"""mortal/train_grp.py on the device: `python -m mortal_b200.train_grp [CONFIG]`, or `train(cfg, steps=None)`.

The loop of the reference's train(), over GrpFileDatasetsIter + grp_loss (mortal_b200.grp_train) instead of a DataLoader, collate
and torch's GRU. It reads the `[grp]` section of the reference's config.toml (the file named on the command line, else
$MORTAL_CFG, else ./config.toml), builds or reads the same file index (`torch.save` of `train_file_list` / `val_file_list`,
reverse-sorted results of recursive globs), keeps the same state file (`model`, `optimizer`, `steps`, `timestamp`) and resumes
from it, and steps torch's `optim.AdamW(grp.parameters())` with its lr overwritten from the config, so state files move between
the two trainers both ways. Every `save_every` steps it runs `val_steps` validation batches forward only, then saves.

Differences from the reference, stated rather than hidden:
- TensorBoard is not used. The scalars the reference writes there (train / val loss and accuracy, lr) go to one `logging` line
  per save instead.
- The reference iterates in a `num_workers=1` DataLoader worker, whose `random` is seeded from torch's RNG. The sample stream here
  is the in-process (`num_workers=0`) stream, so it is not the stream of train_grp.py for a given seed.
"""
from __future__ import annotations

import logging
import os
import sys
import tomllib
from datetime import datetime
from glob import glob
from os import path

import torch
from torch import optim

from .grp_train import GrpFileDatasetsIter, grp_loss
from .model import GRP


def load_config(config_file=None):
    """the whole config.toml as a dict (config.py: MORTAL_CFG, else config.toml)"""
    config_file = config_file or os.environ.get("MORTAL_CFG", "config.toml")
    with open(config_file, "rb") as f:
        return tomllib.load(f)


def _file_lists(ds):
    file_index = ds["file_index"]
    if path.exists(file_index):
        index = torch.load(file_index, weights_only=True)
        return index["train_file_list"], index["val_file_list"]
    logging.info("building file index...")
    train_file_list, val_file_list = [], []
    for pat in ds["train_globs"]:
        train_file_list.extend(glob(pat, recursive=True))
    for pat in ds["val_globs"]:
        val_file_list.extend(glob(pat, recursive=True))
    train_file_list.sort(reverse=True)
    val_file_list.sort(reverse=True)
    torch.save({"train_file_list": train_file_list, "val_file_list": val_file_list}, file_index)
    return train_file_list, val_file_list


def train(cfg, steps=None):
    """train_grp.py train() over `cfg`, the config's `[grp]` table (dict). `steps` bounds this call to that many training steps
    (None: until interrupted, as the reference runs). Returns (grp, optimizer, total steps)."""
    batch_size = cfg["control"]["batch_size"]
    save_every = cfg["control"]["save_every"]
    val_steps = cfg["control"]["val_steps"]
    device = torch.device(cfg["control"]["device"])
    if device.type != "cuda":
        raise ValueError(f"the GRP trainer runs on a CUDA device, got {device}")
    device = torch.device("cuda", device.index if device.index is not None else torch.cuda.current_device())
    logging.info(f"device: {device} ({torch.cuda.get_device_name(device)})")

    grp = GRP(**cfg["network"]).to(device)
    optimizer = optim.AdamW(grp.parameters())
    state_file = cfg["state_file"]
    if path.exists(state_file):
        state = torch.load(state_file, weights_only=True, map_location=device)
        timestamp = datetime.fromtimestamp(state["timestamp"]).strftime("%Y-%m-%d %H:%M:%S")
        logging.info(f"loaded: {timestamp}")
        grp.load_state_dict(state["model"])
        optimizer.load_state_dict(state["optimizer"])
        total = state["steps"]
    else:
        total = 0
    lr = cfg["optim"]["lr"]
    optimizer.param_groups[0]["lr"] = lr

    train_file_list, val_file_list = _file_lists(cfg["dataset"])
    fbs = cfg["dataset"]["file_batch_size"]
    train_data = iter(GrpFileDatasetsIter(train_file_list, fbs, cycle=True, batch_size=batch_size, device=device.index))
    val_data = iter(GrpFileDatasetsIter(val_file_list, fbs, cycle=True, batch_size=batch_size, device=device.index))
    logging.info(f"train file list size: {len(train_file_list):,}")
    logging.info(f"val file list size: {len(val_file_list):,}")
    logging.info(f"total steps: {total:,} est. {total * batch_size / (len(train_file_list) * 10) * 100:6.3f}%")

    zero = lambda: torch.zeros((), dtype=torch.float64, device=device)
    stats = {k: zero() for k in ("train_loss", "train_acc", "val_loss", "val_acc")}
    done = 0
    while steps is None or done < steps:
        batch = next(train_data)
        optimizer.zero_grad(set_to_none=True)
        loss, acc = grp_loss(grp, batch)
        optimizer.step()
        stats["train_loss"] += loss
        stats["train_acc"] += acc
        total += 1
        done += 1
        if total % save_every == 0:
            for _ in range(val_steps):
                loss, acc = grp_loss(grp, next(val_data), backward=False)
                stats["val_loss"] += loss
                stats["val_acc"] += acc
            logging.info(f"steps {total:,}: loss train {(stats['train_loss'] / save_every).item():.6f} "
                         f"val {(stats['val_loss'] / max(val_steps, 1)).item():.6f}, acc train "
                         f"{(stats['train_acc'] / save_every).item():.6f} val {(stats['val_acc'] / max(val_steps, 1)).item():.6f}, "
                         f"lr {lr}")
            for k in stats:
                stats[k] = zero()
            logging.info(f"total steps: {total:,} est. {total * batch_size / (len(train_file_list) * 10) * 100:6.3f}%")
            torch.save({"model": grp.state_dict(), "optimizer": optimizer.state_dict(), "steps": total,
                        "timestamp": datetime.now().timestamp()}, state_file)
    return grp, optimizer, total


def main(argv=None):
    argv = sys.argv[1:] if argv is None else argv
    logging.basicConfig(level=logging.INFO, format="%(asctime)s %(levelname)s %(message)s")
    try:
        train(load_config(argv[0] if argv else None)["grp"])
    except KeyboardInterrupt:
        pass


if __name__ == "__main__":
    main()
