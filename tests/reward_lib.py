"""Helpers of the GRP reward tests — TEST INFRASTRUCTURE: the host build of csrc/mjx_reward.cuh (tests/host_emul/emul_reward.cc)
and a torch-CPU float64 restatement of the reference: model.py GRP (nn.GRU + the FC head + calc_matrix), reward_calculator.py
with the literal prefix-list formulation (pack_padded_sequence over feature[:k+1] for every k), and the per-move loop of
dataloader.py populate_buffer."""
from __future__ import annotations

import ctypes as C
from itertools import permutations

import numpy as np
import torch
from torch import nn
from torch.nn.utils.rnn import pack_padded_sequence, pad_sequence

import emul_lib as E


def emul_lib():
    """emul_lib.lib() with the emulated kernels' entry declared"""
    L = E.lib()
    L.emulr_grp_reward.restype = C.c_int
    L.emulr_grp_reward.argtypes = ([C.c_int, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_int, C.c_int,
                                    C.c_void_p, C.c_int, C.c_void_p, C.c_longlong] + [C.c_void_p] * 8 + [C.c_int]
                                   + [C.c_void_p] * 4)
    return L


# ---------------------------------------------------------------- the reference, restated

class RefGRP(nn.Module):
    """model.py GRP: GRU over the 7 features, Linear HL -> HL, ReLU, Linear HL -> 24, all float64"""

    def __init__(self, hidden_size=64, num_layers=2):
        super().__init__()
        self.rnn = nn.GRU(input_size=7, hidden_size=hidden_size, num_layers=num_layers, batch_first=True)
        self.fc = nn.Sequential(nn.Linear(hidden_size * num_layers, hidden_size * num_layers), nn.ReLU(inplace=True),
                                nn.Linear(hidden_size * num_layers, 24))
        for mod in self.modules():
            mod.to(torch.float64)
        perms = torch.tensor(list(permutations(range(4))))
        self.register_buffer("perms", perms)
        self.register_buffer("perms_t", perms.transpose(0, 1))

    def forward(self, inputs):
        lengths = torch.tensor([t.shape[0] for t in inputs], dtype=torch.int64)
        packed = pack_padded_sequence(pad_sequence(inputs, batch_first=True), lengths, batch_first=True, enforce_sorted=False)
        _, state = self.rnn(packed)
        return self.fc(state.transpose(0, 1).flatten(1))

    def calc_matrix(self, logits):
        probs = logits.softmax(-1)
        matrix = torch.zeros(logits.shape[0], 4, 4, dtype=probs.dtype)
        for player in range(4):
            for rank in range(4):
                matrix[:, player, rank] = probs[:, self.perms_t[player] == rank].sum(-1)
        return matrix


def random_grp(hidden, layers, seed):
    """a RefGRP with random weights, fc.2 scaled up so the softmax is neither flat nor one-hot"""
    torch.manual_seed(seed)
    m = RefGRP(hidden, layers).eval()
    with torch.no_grad():
        for name, p in m.named_parameters():
            p.uniform_(-1.0, 1.0)
            p.mul_((12.0 if name.startswith("fc.2") else 1.0) / np.sqrt(p.shape[-1]))
    return m


def random_feature(n, rng):
    """n kyoku rows as Grp features: grand_kyoku 0..11, honba, kyotaku, scores / 10000 around 2.5 (some tied)"""
    f = np.zeros((n, 7), dtype=np.float64)
    f[:, 0] = np.sort(rng.integers(0, 12, size=n))
    f[:, 1] = rng.integers(0, 6, size=n)
    f[:, 2] = rng.integers(0, 4, size=n)
    sc = rng.integers(-40, 600, size=(n, 4)) * 100
    tie = rng.random(n) < 0.2
    sc[tie, 1] = sc[tie, 0]
    f[:, 3:] = sc / 10000.0
    return f


def ref_calc_grp(grp, feature):
    """reward_calculator.py calc_grp: the net over the list of every prefix"""
    seq = [torch.as_tensor(feature[:i + 1]) for i in range(len(feature))]
    with torch.inference_mode():
        logits = grp(seq)
    return grp.calc_matrix(logits)


def ref_rank_prob(matrix, uniform_init, player_id, rank_by_player):
    """reward_calculator.py calc_rank_prob over calc_grp's matrix"""
    final_ranking = torch.zeros((1, 4))
    final_ranking[0, rank_by_player[player_id]] = 1.
    rank_prob = torch.cat((matrix[:, player_id], final_ranking))
    if uniform_init:
        rank_prob[0, :] = 1 / 4
    return rank_prob


def ref_delta_pt(matrix, pts, uniform_init, player_id, rank_by_player):
    """reward_calculator.py calc_delta_pt over calc_grp's matrix"""
    rank_prob = ref_rank_prob(matrix, uniform_init, player_id, rank_by_player)
    exp_pts = rank_prob @ torch.tensor(pts or [3, 1, -1, -3], dtype=torch.float64)
    return (exp_pts[1:] - exp_pts[:-1]).numpy()


def ref_targets(kyoku_rewards, player_id, feature, final_scores, at_kyoku, dones, apply_gamma):
    """dataloader.py populate_buffer's per-move loop for one Gameplay -> (steps_to_done, kyoku reward, player rank) per move"""
    assert len(kyoku_rewards) >= at_kyoku[-1] + 1
    scores_seq = np.concatenate((feature[:, 3:] * 1e4, [final_scores]))
    player_ranks = (-scores_seq).argsort(-1, kind="stable").argsort(-1, kind="stable")[:, player_id]
    n = len(at_kyoku)
    steps_to_done = np.zeros(n, dtype=np.int64)
    for i in reversed(range(n)):
        if not dones[i]:
            steps_to_done[i] = steps_to_done[i + 1] + int(apply_gamma[i])
    return (steps_to_done, np.array([kyoku_rewards[at_kyoku[i]] for i in range(n)], dtype=np.float64),
            np.array([player_ranks[at_kyoku[i] + 1] for i in range(n)], dtype=np.int64))


# ---------------------------------------------------------------- the emulated kernels

def pack(grp):
    """the weights in mjx_grp_reward_dev's layout (mortal_b200.reward.pack_grp_weights) as numpy"""
    from mortal_b200.reward import pack_grp_weights

    w, h, nl = pack_grp_weights(grp.state_dict())
    return w.numpy(), h, nl


def run_emul(weights, hidden, layers, feats, jobs=None, pts=(3, 1, -1, -3), uniform_init=False, n_rows=None, n_weights=None):
    """emulr_grp_reward -> (rc, matrix [R, 4, 4], steps, reward, rank, status). feats: per-game [L, 7] arrays, or a dict with the
    packed `feat` and `game_off` (hostile-array runs); jobs: dict of move_off, job_game, job_player, at_kyoku, apply_gamma, dones,
    rank, final (numpy); n_rows / n_weights override the counts passed"""
    L = emul_lib()
    if isinstance(feats, dict):
        feat, off = np.ascontiguousarray(feats["feat"], dtype=np.float64), np.ascontiguousarray(feats["game_off"], dtype=np.int32)
    else:
        feat = np.ascontiguousarray(np.concatenate(feats) if feats else np.zeros((0, 7)), dtype=np.float64)
        off = np.zeros(len(feats) + 1, dtype=np.int32)
        np.cumsum([len(f) for f in feats], out=off[1:])
    R = len(feat)
    matrix = np.full((R, 4, 4), np.nan)
    ptr = lambda x: x.ctypes.data if x is not None and x.size else None
    n_jobs = n_moves = 0
    out = [None] * 4
    args = [None] * 8
    if jobs is not None:
        n_jobs, n_moves = len(jobs["job_game"]), int(jobs["n_moves"] if "n_moves" in jobs else jobs["move_off"][-1])
        out = [np.full(n_moves, -7, dtype=np.int64), np.full(n_moves, np.nan), np.full(n_moves, -7, dtype=np.int64),
               np.full(n_jobs, -1, dtype=np.int32)]
        dt = dict(move_off=np.int32, job_game=np.int32, job_player=np.uint8, at_kyoku=np.int32, apply_gamma=np.uint8, dones=np.uint8,
                  rank=np.uint8, final=np.int64)
        args = [np.ascontiguousarray(jobs[k], dtype=v) for k, v in dt.items()]
    p = np.array(pts, dtype=np.float64)
    w = np.ascontiguousarray(weights, dtype=np.float64)
    rc = L.emulr_grp_reward(len(off) - 1, ptr(feat), off.ctypes.data, R if n_rows is None else n_rows, ptr(w),
                            w.size if n_weights is None else n_weights, hidden, layers, ptr(matrix), n_jobs, *[ptr(a) for a in args[:1]],
                            n_moves, *[ptr(a) for a in args[1:]], p.ctypes.data, int(uniform_init), *[ptr(o) for o in out])
    return (rc, matrix, *out)


def jobs_of(gameplays, feats, ranks, finals):
    """the jobs arrays of (player_id, at_kyoku, dones, apply_gamma, game index) tuples"""
    move_off = np.zeros(len(gameplays) + 1, dtype=np.int32)
    np.cumsum([len(g[1]) for g in gameplays], out=move_off[1:])
    cat = lambda i, dt: np.concatenate([np.asarray(g[i], dtype=dt) for g in gameplays]) if gameplays else np.zeros(0, dtype=dt)
    return dict(move_off=move_off, job_game=np.array([g[4] for g in gameplays], dtype=np.int32),
                job_player=np.array([g[0] for g in gameplays], dtype=np.uint8), at_kyoku=cat(1, np.int32), dones=cat(2, np.uint8),
                apply_gamma=cat(3, np.uint8), rank=np.array(ranks, dtype=np.uint8).reshape(-1, 4),
                final=np.array(finals, dtype=np.int64).reshape(-1, 4))


def random_gameplay(n_kyoku, rng, player_id, game):
    """a Gameplay's per-move arrays over a game of n_kyoku rows: (player_id, at_kyoku, dones, apply_gamma, game)"""
    per = rng.integers(0, 12, size=n_kyoku)
    per[-1] = max(per[-1], 1)
    at_kyoku = np.repeat(np.arange(n_kyoku), per).astype(np.int64)
    dones = np.append(at_kyoku[1:] > at_kyoku[:-1], True)
    apply_gamma = rng.random(len(at_kyoku)) < 0.7
    return (player_id, at_kyoku, dones, apply_gamma, game)
