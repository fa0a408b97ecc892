"""Helpers of the GRP training tests — TEST INFRASTRUCTURE: the host build of csrc/mjx_grp_train.cuh
(tests/host_emul/emul_grp_train.cc), and a torch float64 restatement of the reference's train_grp.py step: the batch's prefixes
through pad_sequence + pack_padded_sequence (collate), GRP.forward_packed, get_label, F.cross_entropy and backward(); and its
GrpFileDatasetsIter over stub or real file lists."""
from __future__ import annotations

import ctypes as C
import random

import numpy as np
import torch
from torch.nn import functional as F
from torch.nn.utils.rnn import pack_padded_sequence, pad_sequence

import emul_lib as E
from reward_lib import RefGRP, random_feature, random_grp  # noqa: F401  (re-exported for the tests)


def emul_lib():
    """emul_lib.lib() with the emulated kernels' entries declared"""
    L = E.lib()
    L.emult_grp_train.restype = C.c_int
    L.emult_grp_train.argtypes = ([C.c_int, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_int, C.c_int,
                                   C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 5 + [C.c_int]
                                  + [C.c_void_p] * 5 + [C.c_longlong])
    L.emult_scratch_bytes.restype = C.c_longlong
    L.emult_scratch_bytes.argtypes = [C.c_int] * 5
    return L


def pack(grp):
    """the weights in the packed layout as numpy (the parameters in module order)"""
    return torch.cat([p.detach().reshape(-1) for p in grp.parameters()]).numpy().copy(), grp.rnn.hidden_size, grp.rnn.num_layers


def jobs_of(game, length):
    """the job grouping mortal_b200.grp_train.make_batch builds: dict of int32 arrays and max_steps"""
    game = np.asarray(game, dtype=np.int64)
    job_game, sample_job = np.unique(game, return_inverse=True)
    job_steps = np.zeros(len(job_game), dtype=np.int64)
    np.maximum.at(job_steps, sample_job, np.asarray(length, dtype=np.int64))
    off = np.zeros(len(job_game) + 1, dtype=np.int64)
    np.cumsum(np.bincount(sample_job, minlength=len(job_game)), out=off[1:])
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
    return dict(job_game=i32(job_game), job_steps=i32(job_steps), sample_job=i32(sample_job), job_sample_off=i32(off),
                job_sample=i32(np.argsort(sample_job, kind="stable")), max_steps=int(job_steps.max()) if len(job_steps) else 1)


def run_emul(weights, hidden, layers, feats, game, length, rank, grad=True, jobs=None, n_rows=None, n_weights=None,
             n_samples=None, scratch_bytes=None):
    """emult_grp_train -> (rc, loss, acc, grad [n_weights] (NaN-filled when not written), status [B]). feats: per-game [L, 7]
    arrays or a dict with the packed `feat` and `game_off` (hostile runs); jobs: override of jobs_of(game, length); the other
    keywords override the counts passed"""
    L = emul_lib()
    if isinstance(feats, dict):
        feat, off = np.ascontiguousarray(feats["feat"], dtype=np.float64), np.ascontiguousarray(feats["game_off"], dtype=np.int32)
    else:
        feat = np.ascontiguousarray(np.concatenate(feats), dtype=np.float64)
        off = np.zeros(len(feats) + 1, dtype=np.int32)
        np.cumsum([len(f) for f in feats], out=off[1:])
    game = np.ascontiguousarray(game, dtype=np.int32)
    length = np.ascontiguousarray(length, dtype=np.int32)
    rank = np.ascontiguousarray(rank, dtype=np.int64).reshape(-1, 4)
    B = len(game) if n_samples is None else n_samples
    jb = jobs_of(game, length) if jobs is None else jobs
    J = len(jb["job_game"])
    w = np.ascontiguousarray(weights, dtype=np.float64)
    nb = L.emult_scratch_bytes(hidden, layers, B, J, jb["max_steps"])
    scratch = np.full(max(nb, 8) // 8, np.nan)
    out = np.full(2, np.nan)
    g = np.full(w.size, np.nan)
    status = np.full(max(B, 1), -1, dtype=np.int32)
    ptr = lambda x: x.ctypes.data if x is not None and x.size else None
    rc = L.emult_grp_train(len(off) - 1, ptr(feat), off.ctypes.data, len(feat) if n_rows is None else n_rows, ptr(w),
                           w.size if n_weights is None else n_weights, hidden, layers, B, ptr(game), ptr(length), ptr(rank), J,
                           *[ptr(jb[k]) for k in ("job_game", "job_steps", "sample_job", "job_sample_off", "job_sample")],
                           jb["max_steps"], out.ctypes.data, out[1:].ctypes.data, g.ctypes.data if grad else None, status.ctypes.data,
                           scratch.ctypes.data, nb if scratch_bytes is None else scratch_bytes)
    return rc, out[0], out[1], g, status[:B]


# ---------------------------------------------------------------- the reference, restated

def get_label(rank_by_player):
    """model.py GRP.get_label"""
    perms = RefGRP(1, 1).perms
    B = rank_by_player.shape[0]
    mappings = (perms.expand(B, -1, -1).transpose(0, 1) == rank_by_player).all(-1).nonzero()
    labels = torch.zeros(B, dtype=torch.int64)
    labels[mappings[:, 1]] = mappings[:, 0]
    return labels


def ref_step(grp, inputs, rank, backward=True):
    """train_grp.py's collate + loss step over a list of prefix tensors: (loss, acc) as Python floats; with backward the
    parameters' .grad (zeroed first)"""
    lengths = torch.tensor([len(x) for x in inputs])
    packed = pack_padded_sequence(pad_sequence(inputs, batch_first=True), lengths, batch_first=True, enforce_sorted=False)
    grp.zero_grad(set_to_none=True)
    with torch.set_grad_enabled(backward):
        _, state = grp.rnn(packed)
        logits = grp.fc(state.transpose(0, 1).flatten(1))
        labels = get_label(torch.as_tensor(rank, dtype=torch.int64).to(logits.device))
        loss = F.cross_entropy(logits, labels.to(logits.device))
        acc = (logits.argmax(-1) == labels.to(logits.device)).to(torch.float64).mean()
        if backward:
            loss.backward()
    return loss.item(), acc.item()


def ref_grads(grp):
    return [p.grad.detach().cpu().numpy().reshape(-1).copy() for p in grp.parameters()]


def split(flat, grp):
    out, at = [], 0
    for p in grp.parameters():
        out.append(flat[at:at + p.numel()])
        at += p.numel()
    return out


def grad_err(got_flat, grp):
    """max over the parameters of max |got - ref| / max |ref| (ref = the .grad tensors)"""
    err = 0.0
    for g, r in zip(split(got_flat, grp), ref_grads(grp)):
        err = max(err, np.abs(g - r).max() / max(np.abs(r).max(), 1e-300))
    return err


class RefGrpFileDatasetsIter:
    """train_grp.py GrpFileDatasetsIter restated over a loader `load(file_list) -> list of (feature, rank_by_player)`"""

    def __init__(self, file_list, load, file_batch_size=50, cycle=False):
        self.file_list, self.load, self.file_batch_size, self.cycle = file_list, load, file_batch_size, cycle
        self.buffer = []

    def __iter__(self):
        while True:
            random.shuffle(self.file_list)
            for start_idx in range(0, len(self.file_list), self.file_batch_size):
                for feature, rank_by_player in self.load(self.file_list[start_idx:start_idx + self.file_batch_size]):
                    for i in range(feature.shape[0]):
                        self.buffer.append((torch.as_tensor(feature[:i + 1], dtype=torch.float64), rank_by_player))
                buffer_size = len(self.buffer)
                for i in random.sample(range(buffer_size), buffer_size):
                    yield self.buffer[i]
                self.buffer.clear()
            if not self.cycle:
                break


def ref_batches(it, batch_size, n_batches=None):
    """DataLoader(batch_size, drop_last=True, num_workers=0)'s batching of an iterable: lists of samples"""
    from torch.utils.data import DataLoader, IterableDataset

    class _DS(IterableDataset):
        def __iter__(self):
            return iter(it)

    out = []
    for b in DataLoader(_DS(), batch_size=batch_size, drop_last=True, collate_fn=lambda x: x):
        out.append(b)
        if n_batches is not None and len(out) == n_batches:
            break
    return out
