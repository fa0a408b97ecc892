"""mortal/reward_calculator.py and the per-move targets of mortal/dataloader.py:80-126 on the GPU (csrc/mjx_reward.cuh).

`RewardCalculator(grp, pts=None, uniform_init=False, *, device=0)` is call-compatible with the reference's. The GRP net runs as one
float64 kernel, k_grp_matrix: a GRU starts from h0 = 0 and is causal, so one recurrent pass over a game gives the final hidden
state of every prefix feature[:k+1] (the reference packs all L prefixes, L(L+1)/2 GRU steps). The FC head, the softmax and the
permutation sums of GRP.calc_matrix run behind each step.

`training_samples(data, reward_calc)` is dataloader.py's populate_buffer for a whole `GameplayLoader.load_gz_log_files` /
`load_logs` result: the GRP of every game once (a log's Gameplays share one Grp), then k_train_targets for every Gameplay's moves.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

MAX_HIDDEN, MAX_LAYERS = 256, 4  # include/mjx.h mjx_grp_reward_dev
_GRP_IN = 7
_DEFAULT_PTS = [3, 1, -1, -3]
_TORCH_DTYPE = {np.dtype(np.float64): torch.float64, np.dtype(np.int64): torch.int64, np.dtype(np.int32): torch.int32,
                np.dtype(np.uint8): torch.uint8}


def pack_grp_weights(state):
    """a GRP state dict (model.py GRP: `rnn.*`, `fc.0.*`, `fc.2.*`) -> (float64 CPU tensor in mjx_grp_reward_dev's layout, hidden
    size, layers); ValueError for a shape the kernel does not take (1 <= hidden <= 256, 1 <= layers <= 4, 7 inputs, 24 outputs)"""
    layers = 0
    while f"rnn.weight_ih_l{layers}" in state:
        layers += 1
    if layers == 0 or "rnn.weight_hh_l0" not in state:
        raise ValueError("not a GRP state dict: no rnn.weight_ih_l0 / rnn.weight_hh_l0")
    hidden = int(state["rnn.weight_hh_l0"].shape[1])
    if not (1 <= hidden <= MAX_HIDDEN and 1 <= layers <= MAX_LAYERS):
        raise ValueError(f"unsupported GRP shape: hidden_size {hidden}, num_layers {layers} (supported: hidden_size 1..{MAX_HIDDEN}, "
                         f"num_layers 1..{MAX_LAYERS})")
    hl = hidden * layers
    want = {}
    for k in range(layers):
        want[f"rnn.weight_ih_l{k}"] = (3 * hidden, _GRP_IN if k == 0 else hidden)
        want[f"rnn.weight_hh_l{k}"] = (3 * hidden, hidden)
        want[f"rnn.bias_ih_l{k}"] = (3 * hidden,)
        want[f"rnn.bias_hh_l{k}"] = (3 * hidden,)
    want.update({"fc.0.weight": (hl, hl), "fc.0.bias": (hl,), "fc.2.weight": (24, hl), "fc.2.bias": (24,)})
    for name, shape in want.items():
        if name not in state or tuple(state[name].shape) != shape:
            got = tuple(state[name].shape) if name in state else "missing"
            raise ValueError(f"GRP state dict: {name} is {got}, expected {shape} for hidden_size {hidden}, num_layers {layers}")
    return torch.cat([torch.as_tensor(state[n]).detach().to("cpu", torch.float64).reshape(-1) for n in want]), hidden, layers


def _upload(arrays, dev):
    """numpy arrays -> device tensors of the same dtypes and shapes, with one host-to-device copy (each 8-byte aligned in one
    buffer)"""
    arrays = [np.ascontiguousarray(a) for a in arrays]
    offs = np.concatenate([[0], np.cumsum([(a.nbytes + 7) // 8 * 8 for a in arrays])]).astype(np.int64)
    buf = np.zeros(int(offs[-1]), dtype=np.uint8)
    for a, o in zip(arrays, offs):
        buf[o:o + a.nbytes] = a.reshape(-1).view(np.uint8)
    d = torch.from_numpy(buf).to(dev)
    return [d[o:o + a.nbytes].view(_TORCH_DTYPE[a.dtype]).reshape(a.shape) for a, o in zip(arrays, offs)]


def _feature(f):
    f = np.asarray(f, dtype=np.float64)
    if f.ndim != 2 or f.shape[1] != _GRP_IN or f.shape[0] == 0:
        raise ValueError(f"a GRP feature is float64 [n_kyoku >= 1, 7], got shape {f.shape}")
    return f


class RewardCalculator:
    """mortal/reward_calculator.py on `device` (cuda:`device`, whatever torch's current device is). `grp` is a GRP nn.Module or its
    state dict (`grp_state['model']`); its weights are packed to the device once, here, so later changes to the module are not
    seen. Differences from the reference, stated rather than hidden: `calc_grp` and `calc_rank_prob` return float64 CUDA tensors
    (the reference's are CPU tensors); `calc_delta_pt_batch` is new."""

    def __init__(self, grp, pts=None, uniform_init=False, *, device=0):
        self.device = torch.device("cuda", device)
        state = grp.state_dict() if isinstance(grp, torch.nn.Module) else grp
        w, self.hidden, self.layers = pack_grp_weights(state)
        self.uniform_init = uniform_init
        pts = pts or _DEFAULT_PTS
        if len(pts) != 4:
            raise ValueError(f"pts must have 4 entries, got {len(pts)}")
        self.pts = torch.tensor(pts, dtype=torch.float64)
        self._pts_host = (C.c_double * 4)(*[float(p) for p in pts])
        self.weights = w.to(self.device)

    def _launch(self, feats, jobs=None):
        """mjx_grp_reward_dev over the games' features (and the jobs: a dict of per-job / per-move / per-game numpy arrays)
        -> (matrix [R, 4, 4], (steps_to_done, kyoku_reward, player_rank, job_status) or None), enqueued on the current stream"""
        L = _lib.load()
        dev = self.device
        off = np.zeros(len(feats) + 1, dtype=np.int32)
        np.cumsum([len(f) for f in feats], out=off[1:])
        host = [np.concatenate(feats), off]
        if jobs is not None:
            host += [jobs[k] for k in ("move_off", "job_game", "job_player", "at_kyoku", "apply_gamma", "dones", "rank", "final")]
        d = _upload(host, dev)
        n_rows = int(off[-1])
        matrix = torch.empty((n_rows, 4, 4), dtype=torch.float64, device=dev)
        ptr = lambda t: t.data_ptr() if t is not None and t.numel() else None
        n_jobs = n_moves = 0
        outs = [None] * 4
        args = [None] * 8
        if jobs is not None:
            n_jobs, n_moves = len(jobs["job_game"]), int(jobs["move_off"][-1])
            outs = [torch.empty(n_moves, dtype=torch.int64, device=dev), torch.empty(n_moves, dtype=torch.float64, device=dev),
                    torch.empty(n_moves, dtype=torch.int64, device=dev), torch.empty(n_jobs, dtype=torch.int32, device=dev)]
            args = d[2:]
        mo, jg, jp, ak, ag, dn, rk, fs = (ptr(a) for a in args)
        _lib.check(L.mjx_grp_reward_dev(len(feats), ptr(d[0]), d[1].data_ptr(), n_rows, self.weights.data_ptr(), self.weights.numel(),
                                        self.hidden, self.layers, ptr(matrix), n_jobs, mo, n_moves, jg, jp, ak, ag, dn, rk, fs,
                                        self._pts_host, int(bool(self.uniform_init)), ptr(outs[0]), ptr(outs[1]), ptr(outs[2]),
                                        ptr(outs[3]), torch.cuda.current_stream(dev).cuda_stream), "mjx_grp_reward_dev")
        return matrix, (outs if jobs is not None else None)

    def calc_grp(self, grp_feature):
        """GRP.calc_matrix of every prefix of the game: float64 CUDA [L, 4, 4] (the reference returns a CPU tensor)"""
        with torch.cuda.device(self.device):
            return self._launch([_feature(grp_feature)])[0]

    def calc_rank_prob(self, player_id, grp_feature, rank_by_player):
        """[matrix[:, player_id]; one_hot(rank_by_player[player_id])], row 0 = 1/4 with uniform_init: float64 CUDA [L + 1, 4]"""
        matrix = self.calc_grp(grp_feature)
        final_ranking = torch.zeros((1, 4), dtype=torch.float64, device=self.device)
        final_ranking[0, rank_by_player[player_id]] = 1.
        rank_prob = torch.cat((matrix[:, player_id], final_ranking))
        if self.uniform_init:
            rank_prob[0, :] = 1 / 4
        return rank_prob

    def _delta_pt(self, player_ids, features, ranks, finals):
        """one launch: every game's rewards for its player (a job per game whose moves are its kyoku) -> (float64 CUDA [sum L],
        int64 offsets [G + 1])"""
        feats = [_feature(f) for f in features]
        lens = np.array([len(f) for f in feats], dtype=np.int64)
        move_off = np.zeros(len(feats) + 1, dtype=np.int32)
        np.cumsum(lens, out=move_off[1:])
        n = int(move_off[-1])
        players = np.asarray(player_ids, dtype=np.int64).reshape(-1)
        if len(players) != len(feats) or (players < 0).any() or (players > 3).any():
            raise ValueError("one player id in 0..3 per game")
        jobs = dict(move_off=move_off, job_game=np.arange(len(feats), dtype=np.int32), job_player=players.astype(np.uint8),
                    at_kyoku=np.concatenate([np.arange(k, dtype=np.int32) for k in lens]), apply_gamma=np.zeros(n, dtype=np.uint8),
                    dones=np.ones(n, dtype=np.uint8), rank=np.array(ranks, dtype=np.uint8).reshape(-1, 4),
                    final=np.array(finals, dtype=np.int64).reshape(-1, 4))
        with torch.cuda.device(self.device):
            _, (_, reward, _, status) = self._launch(feats, jobs)
            if (status != 0).any():
                raise RuntimeError(f"mjx_grp_reward_dev: job statuses {status.cpu().numpy().tolist()}")
        return reward, torch.from_numpy(move_off.astype(np.int64))

    def calc_delta_pt(self, player_id, grp_feature, rank_by_player):
        """exp_pts[1:] - exp_pts[:-1] over exp_pts = calc_rank_prob(...) @ pts: numpy float64 [L]"""
        return self._delta_pt([player_id], [grp_feature], [list(rank_by_player)], [[0, 0, 0, 0]])[0].cpu().numpy()

    def calc_delta_pt_batch(self, player_ids, grps):
        """calc_delta_pt of many games in one launch (e.g. over arena.last_grp): game i's rewards for seat player_ids[i] are
        rewards[offsets[i]:offsets[i + 1]] -> (rewards float64 CUDA, offsets int64 CPU tensor [len(grps) + 1])"""
        grps = list(grps)
        if not grps:
            return torch.zeros(0, dtype=torch.float64, device=self.device), torch.zeros(1, dtype=torch.int64)
        return self._delta_pt(player_ids, [g.take_feature() for g in grps], [g.take_rank_by_player() for g in grps],
                              [g.take_final_scores() for g in grps])

    def calc_delta_points(self, player_id, grp_feature, final_scores):
        seq = np.concatenate((grp_feature[:, 3 + player_id] * 1e4, [final_scores[player_id]]))
        delta_points = seq[1:] - seq[:-1]
        return delta_points


def gameplay_targets(data, reward_calc: RewardCalculator):
    """the per-move targets of dataloader.py populate_buffer over a whole GameplayLoader result, in buffer order (file, then
    Gameplay, then move) -> (the Gameplays with moves, dict of device tensors on reward_calc.device: actions int64 [N], masks bool
    [N, 46], steps_to_done int64 [N], kyoku_rewards float64 [N], player_ranks int64 [N]). The GRP runs once per game (a log's
    Gameplays share its Grp). Raises the reference's AssertionError where a Gameplay's at_kyoku[-1] + 1 exceeds its game's kyoku
    count."""
    dev = reward_calc.device
    gps = [gp for file in data for gp in file]
    games, slot, feats = [], {}, []
    jobs, job_game, job_player, counts = [], [], [], []
    for gp in gps:
        at_kyoku = gp._at_kyoku
        if len(at_kyoku) == 0:
            continue
        grp = gp.take_grp()
        g = slot.get(id(grp))
        if g is None:
            g = slot[id(grp)] = len(games)
            games.append(grp)
            feats.append(_feature(grp.take_feature()))
        assert len(feats[g]) >= int(at_kyoku[-1]) + 1  # usually they are equal, unless there is no action in the last kyoku
        jobs.append(gp); job_game.append(g); job_player.append(gp.take_player_id()); counts.append(len(at_kyoku))
    with torch.cuda.device(dev):
        if not jobs:
            z = torch.zeros(0, dtype=torch.int64, device=dev)
            return jobs, dict(actions=z, masks=torch.zeros((0, 46), dtype=torch.bool, device=dev), steps_to_done=z.clone(),
                              kyoku_rewards=torch.zeros(0, dtype=torch.float64, device=dev), player_ranks=z.clone())
        move_off = np.zeros(len(jobs) + 1, dtype=np.int32)
        np.cumsum(counts, out=move_off[1:])
        host = dict(move_off=move_off, job_game=np.array(job_game, dtype=np.int32), job_player=np.array(job_player, dtype=np.uint8),
                    at_kyoku=np.concatenate([gp._at_kyoku for gp in jobs]).astype(np.int32),
                    apply_gamma=np.concatenate([gp._apply_gamma for gp in jobs]).astype(np.uint8),
                    dones=np.concatenate([gp._dones for gp in jobs]).astype(np.uint8),
                    rank=np.array([g.take_rank_by_player() for g in games], dtype=np.uint8),
                    final=np.array([g.take_final_scores() for g in games], dtype=np.int64))
        _, (steps, reward, rank, status) = reward_calc._launch(feats, host)
        out = dict(actions=torch.from_numpy(np.concatenate([np.asarray(gp._actions, dtype=np.int64) for gp in jobs])).to(dev),
                   masks=torch.cat([gp.take_masks().to(dev) for gp in jobs]), steps_to_done=steps, kyoku_rewards=reward,
                   player_ranks=rank)
        if (status != 0).any():
            raise RuntimeError(f"mjx_grp_reward_dev: job statuses {status.cpu().numpy().tolist()}")
    return jobs, out


def training_samples(data, reward_calc: RewardCalculator):
    """dataloader.py populate_buffer over a whole GameplayLoader result (list per file of list of Gameplay): the buffer's entries
    before its shuffle (file, then Gameplay, then move) as device tensors on reward_calc.device, a dict of
        obs            float32 [N, C, 34]
        invisible_obs  float32 [N, C', 34], only when the loader had oracle=True (and some Gameplay has moves)
        actions        int64 [N]
        masks          bool [N, 46]
        steps_to_done  int64 [N]
        kyoku_rewards  float64 [N]
        player_ranks   int64 [N]
    with the targets of gameplay_targets. A Gameplay with no moves contributes no samples (the reference fails on it with an
    IndexError)."""
    dev = reward_calc.device
    jobs, targets = gameplay_targets(data, reward_calc)
    oracle = bool(jobs) and all(gp._invisible is not None for gp in jobs)
    with torch.cuda.device(dev):
        cat = lambda xs: torch.cat([x.to(dev) for x in xs]) if xs else torch.zeros((0, 0, 34), device=dev)
        out = dict(obs=cat([gp.take_obs() for gp in jobs]))
        if oracle:
            out["invisible_obs"] = cat([gp.take_invisible_obs() for gp in jobs])
    out.update(targets)
    return out
