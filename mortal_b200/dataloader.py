"""mortal/dataloader.py FileDatasetsIter with its shuffle buffer on the GPU, yielding batches.

`FileDatasetsIter(version, file_list, pts, oracle=False, file_batch_size=20, reserve_ratio=0, player_names=None, excludes=None,
num_epochs=1, enable_augmentation=False, augmented_first=False, *, grp, batch_size, trust_seed=False, device=0)` yields
`(obs, actions, masks, steps_to_done, kyoku_rewards, player_ranks)` batches (with `oracle=True`, `invisible_obs` after `obs`):
sample for sample what `DataLoader(<the reference's FileDatasetsIter>, batch_size=batch_size)` yields for the same state of
Python's `random` module, which it consumes with the same `random.shuffle` calls in the same order. Batches are fresh CUDA tensors
on cuda:`device`: float32 obs / invisible_obs, int64 actions, bool masks, int64 steps_to_done, float64 kyoku_rewards, int64
player_ranks.

The buffer keeps each observation as a lossless record (include/mjx.h mjx_obs_pack_dev: a 64-bit column mask per row plus the
rows that hold other values than 0 / 1; 19,112 bytes instead of 137,632 for a v4 observation) packed straight from the loader's
tensors, and the other columns as device tensors. A batch is turned back into float32 by one gather kernel (mjx_obs_unpack_dev).
Nothing crosses PCIe per sample. Which samples come out in which batch is decided by `batch_schedule` alone, over the sample
count of every file batch; the device code only moves records.
"""
from __future__ import annotations

import random

import numpy as np
import torch

from . import _lib
from .dataset import GameplayLoader
from .reward import RewardCalculator, gameplay_targets

# bytes a buffered sample keeps beside its observation records: actions, steps_to_done, kyoku_rewards, player_ranks (8 each), masks
COLUMN_BYTES = 4 * 8 + 46
_COLUMNS = ("actions", "masks", "steps_to_done", "kyoku_rewards", "player_ranks")


def batch_schedule(passes, reserve_ratio, batch_size):
    """The sample order of the reference's FileDatasetsIter under DataLoader(batch_size, drop_last=False), over sample ids: the
    samples of the whole run are numbered 0, 1, ... in load order (pass, file batch, then populate_buffer's order).

    `passes` is an iterable of load_files passes, each an iterable of per-file-batch sample counts. Both are consumed lazily, at
    the point where the reference would load that file batch, so a pass can do its own `random.shuffle(file_list)` when it is
    started and load a file batch when its count is asked for. Yields each batch as a list of sample ids, as soon as the reference
    would have collated it; the last batch may be short. Calls `random.shuffle` exactly where the reference does, on lists of the
    same lengths."""
    if batch_size <= 0:
        raise ValueError(f"batch_size must be positive, got {batch_size}")
    next_id = 0
    pending = []
    for counts in passes:
        buffer = []
        for n in counts:
            old_size = len(buffer)
            buffer.extend(range(next_id, next_id + n))
            next_id += n
            reserved_size = int((len(buffer) - old_size) * reserve_ratio)
            if reserved_size > len(buffer):
                continue
            random.shuffle(buffer)
            pending.extend(buffer[reserved_size:])
            del buffer[reserved_size:]
            while len(pending) >= batch_size:
                yield pending[:batch_size]
                del pending[:batch_size]
        random.shuffle(buffer)
        pending.extend(buffer)
        while len(pending) >= batch_size:
            yield pending[:batch_size]
            del pending[:batch_size]
    if pending:
        yield pending


def obs_record_bytes(version: int, invisible: bool = False) -> int:
    """bytes of one observation record (include/mjx.h mjx_obs_record_bytes)"""
    rb = _lib.load().mjx_obs_record_bytes(version, int(invisible))
    _lib.check(min(rb, 0), "mjx_obs_record_bytes")
    return rb


def pack_obs(obs, version: int, invisible: bool = False, out=None):
    """float32 CUDA observations [n, rows, 34] (rows and columns contiguous; any sample stride) -> (records uint8 [n, record_bytes],
    status int32 [n]: 0, or 1 + the first row that holds a cell other than +0.0 / 1.0 outside the value rows), on obs's device
    and current stream; `out` = (records, status) to write into"""
    L = _lib.load()
    rb = obs_record_bytes(version, invisible)
    n = obs.shape[0]
    if out is None:
        out = (torch.empty((n, rb), dtype=torch.uint8, device=obs.device), torch.empty(n, dtype=torch.int32, device=obs.device))
    rec, status = out
    if rec.shape != (n, rb) or rec.dtype != torch.uint8 or not rec.is_contiguous() or status.shape != (n,) or status.dtype != torch.int32:
        raise ValueError("pack_obs: out must be (uint8 [n, record_bytes], int32 [n]), contiguous")
    if n:
        if obs.dtype != torch.float32 or obs.dim() != 3 or obs.shape[2] != 34 or obs.stride(2) != 1 or obs.stride(1) != 34:
            raise ValueError(f"pack_obs: float32 [n, rows, 34] with contiguous rows expected, got {obs.dtype} {tuple(obs.shape)} "
                             f"strides {obs.stride()}")
        _lib.check(L.mjx_obs_pack_dev(version, int(invisible), n, obs.data_ptr(), obs.stride(0), rec.data_ptr(), status.data_ptr(),
                                      torch.cuda.current_stream(obs.device).cuda_stream), "mjx_obs_pack_dev")
    return rec, status


def unpack_obs(records, idx, version: int, invisible: bool = False):
    """records uint8 CUDA [n_records, record_bytes], idx int64 CUDA [B] -> float32 [B, rows, 34], observation idx[b] in row b"""
    L = _lib.load()
    rows = _lib.load().mjx_oracle_obs_rows(version) if invisible else L.mjx_obs_rows(version)
    idx = idx.to(torch.int64).contiguous()
    out = torch.empty((idx.numel(), rows, 34), dtype=torch.float32, device=records.device)
    if idx.numel():
        _lib.check(L.mjx_obs_unpack_dev(version, int(invisible), records.data_ptr() if records.numel() else None, records.shape[0],
                                        idx.data_ptr(), idx.numel(), out.data_ptr(),
                                        torch.cuda.current_stream(records.device).cuda_stream), "mjx_obs_unpack_dev")
    return out


def _runs(views):
    """group [n_k, rows, 34] views into runs that are consecutive slices of one tensor (same sample stride): one pack launch each
    -> list of (first view, total samples)"""
    runs = []
    for v in views:
        if runs:
            first, n = runs[-1]
            if (v.stride() == first.stride() and v.untyped_storage().data_ptr() == first.untyped_storage().data_ptr()
                    and v.data_ptr() == first.data_ptr() + n * first.stride(0) * 4):
                runs[-1] = (first, n + v.shape[0])
                continue
        runs.append((v, v.shape[0]))
    return runs


class FileDatasetsIter:
    """mortal/dataloader.py FileDatasetsIter on the GPU, yielding batches (module docstring). `grp` is the GRP module or its state
    dict (`grp_state['model']`), for RewardCalculator; `trust_seed` goes to the GameplayLoader (with oracle=True, True keeps the
    loader on the device). `file_list` is shuffled in place, as in the reference. `buffered` is the number of samples held on the
    device (the shuffle buffer, plus the samples batched since the last file batch was loaded: their rows go at the next load),
    `record_bytes` what each of them takes (observation records and the other columns), `buffer_bytes` their product."""

    def __init__(self, version, file_list, pts, oracle=False, file_batch_size=20, reserve_ratio=0, player_names=None, excludes=None,
                 num_epochs=1, enable_augmentation=False, augmented_first=False, *, grp, batch_size, trust_seed=False, device=0):
        if batch_size <= 0:
            raise ValueError(f"batch_size must be positive, got {batch_size}")
        self.version = version
        self.file_list = file_list
        self.pts = pts
        self.oracle = oracle
        self.file_batch_size = file_batch_size
        self.reserve_ratio = reserve_ratio
        self.player_names = player_names
        self.excludes = excludes
        self.num_epochs = num_epochs
        self.enable_augmentation = enable_augmentation
        self.augmented_first = augmented_first
        self.grp = grp
        self.batch_size = batch_size
        self.trust_seed = trust_seed
        self.device = torch.device("cuda", device)
        self.record_bytes = obs_record_bytes(version) + (obs_record_bytes(version, True) if oracle else 0) + COLUMN_BYTES
        self.iterator = None
        self._store = None  # dict of device tensors, one row per buffered sample
        self._ids = np.zeros(0, dtype=np.int64)  # the sample id of every store row, ascending
        self._alive = np.zeros(0, dtype=bool)  # whether the row's sample has not been batched yet
        self._loaded = 0  # samples loaded so far (the next sample id)

    @property
    def buffered(self) -> int:
        return len(self._ids)

    @property
    def buffer_bytes(self) -> int:
        return self.buffered * self.record_bytes

    def build_iter(self):
        self.reward_calc = RewardCalculator(self.grp, self.pts, device=self.device.index)

        def passes():
            for _ in range(self.num_epochs):
                yield self._load_files(self.augmented_first)
                if self.enable_augmentation:
                    yield self._load_files(not self.augmented_first)

        for ids in batch_schedule(passes(), self.reserve_ratio, self.batch_size):
            yield self._batch(ids)
        self._store, self._ids, self._alive = None, self._ids[:0], self._alive[:0]

    def _load_files(self, augmented):
        random.shuffle(self.file_list)
        self.loader = GameplayLoader(self.version, oracle=self.oracle, player_names=self.player_names, excludes=self.excludes,
                                     trust_seed=self.trust_seed, augmented=augmented, device=self.device.index)
        for start_idx in range(0, len(self.file_list), self.file_batch_size):
            yield self._populate(self.file_list[start_idx:start_idx + self.file_batch_size])

    def _load(self, file_list):
        """the Gameplays of a file batch (GameplayLoader.load_gz_log_files)"""
        return self.loader.load_gz_log_files(file_list)

    def _populate(self, file_list):
        """load a file batch into the store (keeping the rows not batched yet) -> its sample count"""
        data = self._load(file_list)
        dev = self.device
        with torch.cuda.device(dev):
            jobs, new = gameplay_targets(data, self.reward_calc)
            n = sum(len(gp._at_kyoku) for gp in jobs)
            kinds = [("obs", False, lambda gp: gp.take_obs())]
            if self.oracle:
                kinds.append(("invisible_obs", True, lambda gp: gp.take_invisible_obs()))
            for key, invisible, take in kinds:
                rec = torch.empty((n, obs_record_bytes(self.version, invisible)), dtype=torch.uint8, device=dev)
                status = torch.empty(n, dtype=torch.int32, device=dev)
                at = 0
                for first, m in _runs([take(gp) for gp in jobs]):
                    view = first.as_strided((m,) + tuple(first.shape[1:]), first.stride())
                    pack_obs(view, self.version, invisible, out=(rec[at:at + m], status[at:at + m]))
                    at += m
                bad = torch.nonzero(status).flatten()
                if bad.numel():
                    self._raise_lossy(file_list, data, jobs, key, int(bad[0]), int(status[bad[0]]))
                new[key] = rec
            # the rows still to be batched, then the new file batch
            keep = np.nonzero(self._alive)[0]
            if self._store is None:
                self._store = new
            else:
                kidx = torch.from_numpy(keep).to(dev)
                self._store = {k: torch.cat([self._store[k].index_select(0, kidx), new[k]]) for k in new}
            self._ids = np.concatenate([self._ids[keep], np.arange(self._loaded, self._loaded + n, dtype=np.int64)])
            self._alive = np.ones(len(self._ids), dtype=bool)
            self._loaded += n
        return n

    def _raise_lossy(self, file_list, data, jobs, key, sample, status):
        start = 0
        for gp in jobs:
            m = len(gp._at_kyoku)
            if sample < start + m:
                break
            start += m
        fi = next(k for k, file in enumerate(data) if any(g is gp for g in file))
        raise ValueError(f"{file_list[fi]}: player {gp.take_player_id()}, move {sample - start}: {key} row {status - 1} holds a "
                         "value other than 0 / 1 outside the value rows of the record layout; it cannot be buffered losslessly")

    def _batch(self, ids):
        slots = np.searchsorted(self._ids, ids)
        self._alive[slots] = False
        dev = self.device
        with torch.cuda.device(dev):
            idx = torch.from_numpy(slots).to(dev)
            S = self._store
            out = [unpack_obs(S["obs"], idx, self.version)]
            if self.oracle:
                out.append(unpack_obs(S["invisible_obs"], idx, self.version, True))
            out += [S[k].index_select(0, idx) for k in _COLUMNS]
        return tuple(out)

    def __iter__(self):
        if self.iterator is None:
            self.iterator = self.build_iter()
        return self.iterator
