"""Data-parallel training's host side (no GPU): the file-list shard rule against the reference's worker_init_fn split, the empty
shard, the test play's seed blocks, and the configurations a data-parallel train() / train_online() refuses."""
from __future__ import annotations

import numpy as np
import pytest

torch = pytest.importorskip("torch")


def worker_init_split(file_list, worker_id, num_workers):
    """mortal/dataloader.py:133-139, restated"""
    per_worker = int(np.ceil(len(file_list) / num_workers))
    start = worker_id * per_worker
    return file_list[start:start + per_worker]


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_shards_follow_worker_init_fn(world):
    from mortal_b200.train import check_shards, shard

    for n in sorted({m * world + d for m in range(1, 5) for d in (-1, 0, 1)} - {0}):
        files = [f"f{i}" for i in range(n)]
        shards = [shard(files, r, world) for r in range(world)]
        assert shards == [worker_init_split(files, r, world) for r in range(world)], n
        assert sum(shards, []) == files, n  # disjoint, contiguous, in order, covering the list
        if all(shards):
            check_shards(n, world)
        else:
            with pytest.raises(ValueError, match="shard"):
                check_shards(n, world)


def test_empty_shard_raises():
    from mortal_b200.train import check_shards

    check_shards(4, 4)
    for n, world in ((5, 4), (1, 2), (0, 2), (6, 4)):  # ceil(5 / 4) = 2 leaves rank 3 nothing; ceil(6 / 4) = 2 too
        with pytest.raises(ValueError, match="shard"):
            check_shards(n, world)


@pytest.mark.parametrize("world", [1, 2, 3, 4, 7])
def test_seed_blocks_cover_every_seed_once(world):
    from mortal_b200.dist import seed_block

    for seeds in range(0, 3 * world + 2):
        covered = []
        for r in range(world):
            start, count = seed_block(seeds, r, world)
            assert count in (seeds // world, seeds // world + 1)
            covered += range(start, start + count)
        assert covered == list(range(seeds)), seeds


def _cfg(batch_size=512, test_device="cuda:0", **control):
    return {"control": {"version": 4, "online": False, "save_every": 2, "opt_step_every": 1, "test_every": 4,
                        "batch_size": batch_size, "device": "cuda:0", **control},
            "resnet": {"conv_channels": 192, "num_blocks": 40},
            "baseline": {"test": {"device": test_device}}}


def test_data_parallel_rejections(monkeypatch):
    from mortal_b200 import train as T

    T.check_config(_cfg(), world=2)
    T.check_config(_cfg(batch_size=510), world=1)
    with pytest.raises(ValueError, match="batch_size = 510"):
        T.check_config(_cfg(batch_size=510), world=4)
    with pytest.raises(ValueError, match=r"\[baseline.test\] device"):
        T.check_config(_cfg(test_device="cuda:1"), world=2)
    T.check_config(_cfg(test_device="cuda:1"), world=1)
    with pytest.raises(ValueError, match="not data-parallel"):
        T.check_online_config({"control": {"online": True}}, world=2)
    # train() and train_online() read the rank count of the initialised default group
    monkeypatch.setattr(T, "world_info", lambda: (None, 0, 3))
    with pytest.raises(ValueError, match="batch_size = 512"):
        T.train(_cfg())
    with pytest.raises(ValueError, match="not data-parallel"):
        T.train_online({"control": {"online": True}})
