"""GRP training on the GPU: mortal/train_grp.py's GrpFileDatasetsIter, collate and loss step (csrc/mjx_grp_train.cuh).

`GrpFileDatasetsIter(file_list, file_batch_size=50, cycle=False, *, batch_size, device=0)` yields `GrpBatch`es: sample for sample
the batches `DataLoader(<the reference's GrpFileDatasetsIter>, batch_size, drop_last=True, collate_fn=collate)` gives for the
same state of Python's `random` module (num_workers=0), which it consumes with the same calls in the same order. A sample is a
game prefix feature[:len] with the game's rank_by_player; a batch holds the kyoku rows of the games it draws from, uploaded once
per file batch, and each sample as (game, len), never as a copied prefix.

`grp_loss(grp, batch, backward=True)` is `F.cross_entropy(grp.forward_packed(inputs), grp.get_label(rank))`, its accuracy, and
`loss.backward()` in one launch sequence: a GRU is causal and starts from h0 = 0, so every prefix of a game is one pass over the
game, forward and backward (about L GRU steps per game and direction where the reference's packed prefixes take L(L+1)/2).
"""
from __future__ import annotations

import random
from typing import NamedTuple

import numpy as np
import torch

from . import _lib
from .dataset import Grp
from .reward import _upload

_GRP_IN = 7


def grp_batch_schedule(passes, batch_size):
    """The sample order of the reference's GrpFileDatasetsIter under DataLoader(batch_size, drop_last=True), over sample ids: the
    samples of the whole run are numbered 0, 1, ... in load order (pass, file batch, then populate_buffer's order: games in file
    order, prefixes ascending).

    `passes` is an iterable of cycles (one for cycle=False), each an iterable of per-file-batch buffer sizes. Both are consumed
    lazily, where the reference would start the cycle (its `random.shuffle(file_list)` belongs to the pass) and load the file
    batch. Yields each full batch as a list of sample ids as soon as the reference would have collated it; a short last batch
    is dropped. Calls `random.sample(range(n), n)` exactly where the reference does."""
    if batch_size <= 0:
        raise ValueError(f"batch_size must be positive, got {batch_size}")
    next_id = 0
    pending = []
    for sizes in passes:
        for n in sizes:
            pending.extend(next_id + i for i in random.sample(range(n), n))
            next_id += n
            while len(pending) >= batch_size:
                yield pending[:batch_size]
                del pending[:batch_size]


class GrpBatch(NamedTuple):
    """One training batch on the device. feat float64 [R, 7]: the kyoku rows of the batch's games, game g at rows
    [game_off[g], game_off[g + 1]) (game_off int32 [G + 1]); per sample game int32 [B], length int32 [B] (the prefix is
    feat[game_off[game] : game_off[game] + length]) and rank_by_player int64 [B, 4]. `jobs` int32 holds the grouping by game
    that mjx_grp_train_dev takes (job_game, job_steps [n_jobs], sample_job [B], job_sample_off [n_jobs + 1], job_sample [B]);
    n_jobs and max_steps are its host-side counts."""
    feat: torch.Tensor
    game_off: torch.Tensor
    game: torch.Tensor
    length: torch.Tensor
    rank_by_player: torch.Tensor
    jobs: torch.Tensor
    n_jobs: int
    max_steps: int


def make_batch(feat, game_lengths, game, length, rank_by_player, device=0):
    """a GrpBatch from the games' rows `feat` (float64 [R, 7], CUDA or host) with per-game row counts `game_lengths` and host
    per-sample arrays game [B], length [B], rank_by_player [B, 4]; validates the samples on the host (ValueError) and uploads the
    index arrays with one copy"""
    dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
    lens = np.asarray(game_lengths, dtype=np.int64).reshape(-1)
    game = np.asarray(game, dtype=np.int64).reshape(-1)
    length = np.asarray(length, dtype=np.int64).reshape(-1)
    rank = np.asarray(rank_by_player, dtype=np.int64)
    B = len(game)
    if B == 0 or len(length) != B or rank.shape != (B, 4):
        raise ValueError(f"a GRP batch needs B >= 1 samples with game [B], length [B], rank_by_player [B, 4]; got {len(game)}, "
                         f"{len(length)}, {rank.shape}")
    if len(lens) == 0 or (lens < 1).any():
        raise ValueError("every game of a GRP batch needs at least one kyoku row")
    if (game < 0).any() or (game >= len(lens)).any():
        raise ValueError(f"sample game index outside 0..{len(lens) - 1}")
    if (length < 1).any() or (length > lens[game]).any():
        raise ValueError("sample prefix length outside 1..its game's kyoku count")
    if tuple(feat.shape) != (int(lens.sum()), _GRP_IN):
        raise ValueError(f"feat must be [{int(lens.sum())}, 7] for these games, got {tuple(feat.shape)}")
    job_game, sample_job = np.unique(game, return_inverse=True)
    job_steps = np.zeros(len(job_game), dtype=np.int64)
    np.maximum.at(job_steps, sample_job, length)
    job_sample = np.argsort(sample_job, kind="stable")
    job_sample_off = np.zeros(len(job_game) + 1, dtype=np.int64)
    np.cumsum(np.bincount(sample_job, minlength=len(job_game)), out=job_sample_off[1:])
    game_off = np.zeros(len(lens) + 1, dtype=np.int64)
    np.cumsum(lens, out=game_off[1:])
    i32 = np.concatenate([game_off, game, length, job_game, job_steps, sample_job, job_sample_off, job_sample]).astype(np.int32)
    d_i32, d_rank = _upload([i32, rank], dev)
    G, J = len(lens), len(job_game)
    cut = np.cumsum([G + 1, B, B])
    if isinstance(feat, np.ndarray):
        feat = _upload([np.ascontiguousarray(feat, dtype=np.float64)], dev)[0]
    elif feat.dtype != torch.float64 or feat.device != dev or not feat.is_contiguous():
        raise ValueError(f"feat must be a contiguous float64 tensor on {dev}")
    return GrpBatch(feat, d_i32[:cut[0]], d_i32[cut[0]:cut[1]], d_i32[cut[1]:cut[2]], d_rank, d_i32[cut[2]:], J,
                    int(job_steps.max()))


class GrpFileDatasetsIter:
    """mortal/train_grp.py GrpFileDatasetsIter + DataLoader(batch_size, drop_last=True, collate_fn=collate) on the device
    (module docstring). `file_list` is shuffled in place, as in the reference. Each file batch is loaded with
    Grp.load_gz_log_files and its kyoku rows uploaded once; its rows stay on the device until all of its samples have been
    batched. `batch_size` may exceed a file batch's buffer: a batch then draws from several file batches."""

    def __init__(self, file_list, file_batch_size=50, cycle=False, *, batch_size, device=0):
        if batch_size <= 0:
            raise ValueError(f"batch_size must be positive, got {batch_size}")
        if file_batch_size <= 0:
            raise ValueError(f"file_batch_size must be positive, got {file_batch_size}")
        self.file_list = file_list
        self.file_batch_size = file_batch_size
        self.cycle = cycle
        self.batch_size = batch_size
        self.device = torch.device("cuda", device)
        self.iterator = None
        self._loaded = 0  # samples loaded so far (the next sample id)
        self._live = []  # file batches with samples not batched yet: dicts of first id, sizes, row offsets, feat, rank, left

    def build_iter(self):
        def passes():
            while True:
                if not self.file_list and self.cycle:
                    raise ValueError("GrpFileDatasetsIter: cycle=True over an empty file list never yields")
                yield self._load_files()
                if not self.cycle:
                    break

        for ids in grp_batch_schedule(passes(), self.batch_size):
            yield self._batch(np.asarray(ids, dtype=np.int64))
        self._live = []

    def _load_files(self):
        random.shuffle(self.file_list)
        for start_idx in range(0, len(self.file_list), self.file_batch_size):
            yield self._populate(self.file_list[start_idx:start_idx + self.file_batch_size])

    def _populate(self, file_list):
        """load a file batch and upload its rows -> its sample count (the sum of its games' kyoku counts)"""
        games = Grp.load_gz_log_files(file_list)
        lens = np.array([len(g.take_feature()) for g in games], dtype=np.int64)
        n = int(lens.sum())
        first = self._loaded
        self._loaded += n
        if n == 0:
            return 0
        keep = [g for g, k in zip(games, lens) if k]
        lens = lens[lens > 0]
        feat = np.concatenate([np.asarray(g.take_feature(), dtype=np.float64) for g in keep])
        with torch.cuda.device(self.device):
            feat_d = _upload([feat], self.device)[0]
        off = np.zeros(len(lens) + 1, dtype=np.int64)
        np.cumsum(lens, out=off[1:])
        self._live.append(dict(first=first, n=n, lens=lens, off=off, feat=feat_d,
                               rank=np.array([g.take_rank_by_player() for g in keep], dtype=np.int64).reshape(-1, 4), left=n))
        return n

    def _batch(self, ids):
        live = self._live
        firsts = np.array([fb["first"] for fb in live], dtype=np.int64)
        which = np.searchsorted(firsts, ids, side="right") - 1
        used = np.unique(which)
        parts = [live[w] for w in used]
        games_before = np.concatenate([[0], np.cumsum([len(fb["lens"]) for fb in parts])])
        game = np.empty(len(ids), dtype=np.int64)
        length = np.empty(len(ids), dtype=np.int64)
        rank = np.empty((len(ids), 4), dtype=np.int64)
        for i, w in enumerate(used):
            fb, sel = live[w], which == w
            local = ids[sel] - fb["first"]
            g = np.searchsorted(fb["off"], local, side="right") - 1
            game[sel] = g + games_before[i]
            length[sel] = local - fb["off"][g] + 1
            rank[sel] = fb["rank"][g]
            fb["left"] -= int(sel.sum())
        with torch.cuda.device(self.device):
            feat = parts[0]["feat"] if len(parts) == 1 else torch.cat([fb["feat"] for fb in parts])
            batch = make_batch(feat, np.concatenate([fb["lens"] for fb in parts]), game, length, rank, self.device)
        self._live = [fb for fb in live if fb["left"] > 0]
        return batch

    def __iter__(self):
        if self.iterator is None:
            self.iterator = self.build_iter()
        return self.iterator


def _grp_shape(grp):
    """(hidden, layers, n_weights) of a GRP module, validated once per module (ValueError for a shape the kernels do not take)"""
    shape = getattr(grp, "_mjx_grp_shape", None)
    if shape is None:
        from .reward import pack_grp_weights

        _, hidden, layers = pack_grp_weights({k: torch.empty(v.shape, dtype=torch.float64) for k, v in grp.state_dict().items()})
        names = [n for n, _ in grp.named_parameters()]
        want = []
        for k in range(layers):
            want += [f"rnn.weight_ih_l{k}", f"rnn.weight_hh_l{k}", f"rnn.bias_ih_l{k}", f"rnn.bias_hh_l{k}"]
        want += ["fc.0.weight", "fc.0.bias", "fc.2.weight", "fc.2.bias"]
        if names != want:
            raise ValueError(f"GRP parameters must be {want} in this order, got {names}")
        if any(p.dtype != torch.float64 or p.device.type != "cuda" for p in grp.parameters()):
            raise ValueError("GRP parameters must be float64 CUDA tensors")
        shape = (hidden, layers, sum(p.numel() for p in grp.parameters()))
        grp._mjx_grp_shape = shape
    return shape


def grp_loss(grp, batch: GrpBatch, backward=True):
    """(loss, acc): float64 CUDA 0-dim tensors equal to F.cross_entropy(logits, labels) and (logits.argmax(-1) ==
    labels).double().mean() of the reference's train_grp.py step. With backward=True every parameter's .grad is left as
    loss.backward() leaves it (created when None, added to otherwise). Enqueued on the current stream; no host synchronise."""
    hidden, layers, n_weights = _grp_shape(grp)
    params = list(grp.parameters())
    dev = params[0].device
    B = int(batch.game.numel())
    if (batch.feat.device != dev or batch.feat.dtype != torch.float64 or batch.feat.dim() != 2 or batch.feat.shape[1] != _GRP_IN
            or batch.rank_by_player.shape != (B, 4) or batch.rank_by_player.dtype != torch.int64 or B == 0
            or batch.length.shape != (B,) or batch.game_off.dtype != torch.int32 or batch.jobs.dtype != torch.int32
            or batch.jobs.numel() != 3 * batch.n_jobs + 2 * B + 1 or not 1 <= batch.n_jobs <= B or batch.max_steps < 1):
        raise ValueError("grp_loss: not a GrpBatch of this device (use make_batch or GrpFileDatasetsIter)")
    L = _lib.load()
    with torch.cuda.device(dev):
        weights = torch.cat([p.detach().reshape(-1) for p in params])
        nb = L.mjx_grp_train_scratch_bytes(hidden, layers, B, batch.n_jobs, batch.max_steps)
        _lib.check(min(nb, 0), "mjx_grp_train_scratch_bytes")
        scratch = torch.empty(nb // 8, dtype=torch.float64, device=dev)
        out = torch.empty(2, dtype=torch.float64, device=dev)
        grad = torch.empty(n_weights, dtype=torch.float64, device=dev) if backward else None
        status = torch.empty(B, dtype=torch.int32, device=dev)
        J = batch.n_jobs
        jobs = batch.jobs
        p = jobs.data_ptr()
        at = lambda k: p + 4 * k
        n_games = int(batch.game_off.numel()) - 1
        _lib.check(L.mjx_grp_train_dev(n_games, batch.feat.data_ptr(), batch.game_off.data_ptr(), batch.feat.shape[0],
                                       weights.data_ptr(), n_weights, hidden, layers, B, batch.game.data_ptr(), batch.length.data_ptr(),
                                       batch.rank_by_player.data_ptr(), J, at(0), at(J), at(2 * J), at(2 * J + B), at(3 * J + B + 1),
                                       batch.max_steps, out.data_ptr(), out[1:].data_ptr(), grad.data_ptr() if backward else None,
                                       status.data_ptr(), scratch.data_ptr(), nb, torch.cuda.current_stream(dev).cuda_stream),
                   "mjx_grp_train_dev")
    if backward:
        at = 0
        for q in params:
            g = grad[at:at + q.numel()].view_as(q)
            at += q.numel()
            if q.grad is None:
                q.grad = g
            else:
                q.grad.add_(g)
    return out[0], out[1]
