"""mortal_b200.dataloader on the device: FileDatasetsIter against the reference's iterator restated (this package's GameplayLoader
and training_samples for populate_buffer, a host list buffer, random.shuffle, torch's DataLoader collation) on 256 arena logs:
every batch equal (observations, invisible observations and masks bitwise, the other columns exactly), dtypes and devices as the
reference collates them, for v4 with and without oracle, v1 and v2, reserve ratios, augmentation, two epochs and batch sizes that
do not divide the stream. Also the device codec against its host build on loader rows, and the buffer statistics."""
import copy
import random

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import obs_pack_lib as P  # noqa: E402
import reward_lib as R  # noqa: E402
from test_gpu_reward import arena_files  # noqa: E402,F401  (module fixture: 256 arena logs)

PTS = [90, 45, 0, -135]


@pytest.fixture(scope="module")
def grp():
    return R.random_grp(64, 2, 21)


class RefIter(torch.utils.data.IterableDataset):
    """mortal/dataloader.py FileDatasetsIter, populate_buffer's entries taken from training_samples (moved to the host, one entry
    per move as the reference builds them)"""

    def __init__(self, version, file_list, oracle, file_batch_size, reserve_ratio, num_epochs, enable_augmentation, augmented_first,
                 trust_seed, grp):
        super().__init__()
        self.version, self.file_list, self.oracle = version, file_list, oracle
        self.file_batch_size, self.reserve_ratio, self.num_epochs = file_batch_size, reserve_ratio, num_epochs
        self.enable_augmentation, self.augmented_first, self.trust_seed = enable_augmentation, augmented_first, trust_seed
        self.grp = grp
        self.iterator = None

    def build_iter(self):
        from mortal_b200.reward import RewardCalculator

        self.reward_calc = RewardCalculator(self.grp, PTS)
        for _ in range(self.num_epochs):
            yield from self.load_files(self.augmented_first)
            if self.enable_augmentation:
                yield from self.load_files(not self.augmented_first)

    def load_files(self, augmented):
        from mortal_b200.dataset import GameplayLoader

        random.shuffle(self.file_list)
        self.loader = GameplayLoader(self.version, oracle=self.oracle, trust_seed=self.trust_seed, augmented=augmented)
        self.buffer = []
        for start_idx in range(0, len(self.file_list), self.file_batch_size):
            old_buffer_size = len(self.buffer)
            self.populate_buffer(self.file_list[start_idx:start_idx + self.file_batch_size])
            buffer_size = len(self.buffer)
            reserved_size = int((buffer_size - old_buffer_size) * self.reserve_ratio)
            if reserved_size > buffer_size:
                continue
            random.shuffle(self.buffer)
            yield from self.buffer[reserved_size:]
            del self.buffer[reserved_size:]
        random.shuffle(self.buffer)
        yield from self.buffer
        self.buffer.clear()

    def populate_buffer(self, file_list):
        from mortal_b200.reward import training_samples

        s = training_samples(self.loader.load_gz_log_files(file_list), self.reward_calc)
        obs = s["obs"].cpu().numpy()
        inv = s["invisible_obs"].cpu().numpy() if self.oracle and "invisible_obs" in s else None
        actions = s["actions"].cpu().numpy().tolist()
        masks = s["masks"].cpu().numpy()
        steps, rewards, ranks = (s[k].cpu().numpy() for k in ("steps_to_done", "kyoku_rewards", "player_ranks"))
        for i in range(len(actions)):
            entry = [obs[i], actions[i], masks[i], steps[i], rewards[i], ranks[i]]
            if self.oracle:
                entry.insert(1, inv[i])
            self.buffer.append(entry)

    def __iter__(self):
        if self.iterator is None:
            self.iterator = self.build_iter()
        return self.iterator


class _OwnRandom:
    """advances an iterator under its own state of Python's `random`, so that two iterators that each consume `random` can be
    stepped in lockstep and each sees the stream it would see alone"""

    def __init__(self, it, state):
        self.it, self.state = it, state

    def __next__(self):
        outer = random.getstate()
        random.setstate(self.state)
        try:
            return next(self.it)
        finally:
            self.state = random.getstate()
            random.setstate(outer)


CASES = [  # (version, oracle, trust_seed, n_files, file_batch_size, reserve_ratio, epochs, augmentation, augmented_first, batch)
    (4, False, False, 256, 20, 0, 1, False, False, 512),
    (4, True, True, 96, 20, 0.5, 1, False, False, 300),
    (1, False, False, 64, 16, 0.5, 1, False, False, 1000),
    (2, False, False, 48, 20, 0, 2, False, False, 777),
    (4, False, False, 48, 12, 0.5, 1, True, True, 512),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"v{c[0]}-oracle{int(c[1])}-r{c[5]}-e{c[6]}-aug{int(c[7])}-b{c[9]}")
def test_iterator_equals_reference(arena_files, grp, case):  # noqa: F811
    from mortal_b200.dataloader import FileDatasetsIter

    version, oracle, trust_seed, n_files, fbs, ratio, epochs, aug, aug_first, bs = case
    files = arena_files[:n_files]
    random.seed(1234 + version)
    ref_files, dev_files = list(files), list(files)
    ref = RefIter(version, ref_files, oracle, fbs, ratio, epochs, aug, aug_first, trust_seed, copy.deepcopy(grp))
    ref_it = _OwnRandom(iter(torch.utils.data.DataLoader(ref, batch_size=bs, drop_last=False, num_workers=0)), random.getstate())
    it = FileDatasetsIter(version, dev_files, PTS, oracle, fbs, ratio, None, None, epochs, aug, aug_first, grp=grp.state_dict(),
                          batch_size=bs, trust_seed=trust_seed)
    assert iter(it) is iter(it)
    dev_it = _OwnRandom(iter(it), random.getstate())
    dev = torch.device("cuda", 0)
    want_dtypes = [torch.float32] * (2 if oracle else 1) + [torch.int64, torch.bool, torch.int64, torch.float64, torch.int64]
    n_batches = n_samples = 0
    peak = None
    while True:
        try:
            w = next(ref_it)
        except StopIteration:
            w = None
        if peak is None:  # the device iterator's first batch: its first file batch loaded, packed and gathered
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            base = torch.cuda.memory_allocated(dev)
        try:
            g = next(dev_it)
        except StopIteration:
            g = None
        if peak is None:
            peak = torch.cuda.max_memory_allocated(dev) - base
        if w is None or g is None:
            assert w is None and g is None, f"stream lengths differ after {n_batches} batches"
            break
        assert len(g) == len(w) == len(want_dtypes)
        for k, (a, b, dt) in enumerate(zip(g, w, want_dtypes)):
            assert a.device == dev and a.dtype == dt == b.dtype and a.shape == b.shape, (n_batches, k, a.dtype, b.dtype, a.shape, b.shape)
            bb = b.to(dev)
            if dt == torch.float32:
                assert torch.equal(a.view(torch.int32), bb.view(torch.int32)), (n_batches, k)
            else:
                assert torch.equal(a, bb), (n_batches, k)
        assert it.buffer_bytes == it.buffered * it.record_bytes and it.buffered > 0
        n_batches += 1
        n_samples += len(g[1 if not oracle else 2])
    assert ref_files == dev_files  # the file list was shuffled in place the same way
    rb = P.record_bytes(version, False) + (P.record_bytes(version, True) if oracle else 0) + 78
    assert it.record_bytes == rb
    assert n_batches == -(-n_samples // bs) and n_samples > 0
    print(f"v{version} oracle={oracle} reserve={ratio} epochs={epochs} aug={aug}: {n_samples} samples in {n_batches} batches equal; "
          f"{rb} B per buffered sample; peak device memory over the first file batch {peak / 2**20:.0f} MiB")


@pytest.mark.parametrize("version,oracle", [(4, True), (1, True), (3, False)])
def test_device_codec_equals_host_build(arena_files, version, oracle):  # noqa: F811
    """k_obs_pack / k_obs_unpack on loader rows against the host build: records, statuses and gathers equal"""
    from mortal_b200.dataloader import pack_obs, unpack_obs
    from mortal_b200.dataset import GameplayLoader

    data = GameplayLoader(version, oracle=oracle, trust_seed=oracle).load_gz_log_files(arena_files[:8])
    gps = [gp for f in data for gp in f if len(gp._at_kyoku)]
    kinds = [(False, gps[0].take_obs(), gps[1].take_obs())] + ([(True, gps[0].take_invisible_obs(), gps[1].take_invisible_obs())]
                                                               if oracle else [])
    for invisible, x0, x1 in kinds:
        for x in (x0, x1, x1[1::3]):  # a Gameplay's slice of the loader tensor, read in place; every third row (a larger pitch)
            rec, status = pack_obs(x, version, invisible)
            h = x.cpu().numpy()
            rc, hrec, hstatus = P.pack(np.ascontiguousarray(h), version, invisible)
            assert rc == 0 and not hstatus.any() and not status.any()
            assert np.array_equal(rec.cpu().numpy(), hrec)
            idx = torch.randint(-2, len(h) + 2, (3 * len(h),), device=x.device)
            y = unpack_obs(rec, idx, version, invisible)
            rc, hy = P.unpack(hrec, idx.cpu().numpy(), version, invisible)
            assert np.array_equal(y.cpu().numpy().view(np.int32), hy.view(np.int32))
        # hostile cells: the same statuses as the host build
        bad = x0.clone()
        vals = set(P.value_rows(version, invisible).tolist())
        rows = [r for r in range(bad.shape[1]) if r not in vals]
        for i, v in zip(range(len(bad)), [0.5, -0.0, float("nan"), 2.0, 1e-45] * len(bad)):
            bad[i, rows[(7 * i) % len(rows)], (5 * i) % 34] = v
        rec, status = pack_obs(bad, version, invisible)
        rc, hrec, hstatus = P.pack(bad.cpu().numpy(), version, invisible)
        assert np.array_equal(status.cpu().numpy(), hstatus) and (hstatus > 0).all()


def test_lossy_observation_raises(arena_files, grp, monkeypatch):  # noqa: F811
    """a cell the record cannot hold names the file, the player and the move"""
    from mortal_b200 import dataloader
    from mortal_b200.dataset import GameplayLoader

    real = GameplayLoader.load_gz_log_files

    def corrupt(self, files):
        data = real(self, files)
        gp = next(gp for f in data for gp in f if len(gp._at_kyoku) > 3)
        gp._obs[3, 0, 0] = 0.5
        return data

    monkeypatch.setattr(GameplayLoader, "load_gz_log_files", corrupt)
    random.seed(0)
    it = dataloader.FileDatasetsIter(4, list(arena_files[:4]), PTS, grp=grp, batch_size=64)
    with pytest.raises(ValueError, match=r"player \d, move 3: obs row 0"):
        next(iter(it))
