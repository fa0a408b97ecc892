"""Self-play games handed to the trainer without their logs: the arena's device event words, converted on the device into the
arrays the replay kernels take (csrc/mjx_selfplay.cuh, include/mjx_selfplay.h).

    arena.record_games = True; arena.py_vs_py(...)        -> arena.last_games, a SelfPlayGames
    decode_games(games, idx, augment)                      -> validate_logs.DecodedLogs (with deltas) of games idx
    GameplayLoader(...).load_games(games, idx)             -> what load_gz_log_files returns for those games' written files
    SelfPlayDatasetsIter(version, games, pts, ...)         -> what dataloader.FileDatasetsIter yields over the written files

The converter makes of every game exactly what the device decoder makes of the text mortal_b200/mjai_log.py writes for it (the
arrays, the line numbers, the deltas; augmented when asked), so the samples are those of the log path by construction, without
rendering, gzip, files or parsing. The start_game event (names, seed) is built on the host from the games' records.
"""
from __future__ import annotations

import os

import numpy as np

from . import _cdecl, _lib
from .dataloader import FileDatasetsIter
from .dataset_codec import HORA_WORDS, KYOKU_WORDS

HEADER = os.path.join(os.path.dirname(_cdecl.HEADER), "mjx_selfplay.h")
with open(HEADER) as _f:
    _TEXT = _f.read()
SYMBOLS = _cdecl.functions(_TEXT, "mjx_arena_words_")  # the entries of include/mjx_selfplay.h, exported by libmjx.so
STATUS = {name.removeprefix("MJX_AW_"): v for name, v in _cdecl.enum(_TEXT, "mjx_aw_status").items()}
_BOUND = None


def _load():
    global _BOUND
    if _BOUND is None:
        _BOUND = _cdecl.bind(_lib.load(), SYMBOLS)
    return _BOUND


class SelfPlayGames:
    """Finished self-play games on the device: words int64 [n, pitch] (the arena's event words, game g's first lens[g] of them valid,
    reads bounded by log_cap), lens int32 [n], and per game the seat names, the (nonce, key) seed, ranks [4] and final scores [4]."""

    def __init__(self, words, lens, log_cap, names, seeds, ranks, scores):
        self.words, self.lens, self.log_cap = words, lens, int(log_cap)
        self.names = [list(x) for x in names]
        self.seeds = [(int(a), int(b)) for a, b in seeds]
        self.ranks = np.asarray(ranks, dtype=np.int64).reshape(-1, 4)
        self.scores = np.asarray(scores, dtype=np.int64).reshape(-1, 4)
        if not (len(self.names) == len(self.seeds) == len(self.ranks) == len(self.scores) == words.shape[0] == lens.shape[0]):
            raise ValueError("SelfPlayGames: one entry per game expected in every field")

    def __len__(self):
        return len(self.seeds)

    @staticmethod
    def concat(parts):
        """the games of several SelfPlayGames, in order (their words must have the same capacity)"""
        import torch

        parts = list(parts)
        if not parts:
            raise ValueError("SelfPlayGames.concat: nothing to concatenate")
        caps = {p.log_cap for p in parts} | {p.words.shape[1] for p in parts}
        if len(caps) != 1:
            raise ValueError(f"SelfPlayGames.concat: the games' log capacities differ ({sorted(caps)})")
        return SelfPlayGames(torch.cat([p.words for p in parts]), torch.cat([p.lens for p in parts]), parts[0].log_cap,
                             [x for p in parts for x in p.names], [x for p in parts for x in p.seeds],
                             np.concatenate([p.ranks for p in parts]), np.concatenate([p.scores for p in parts]))

    def first_event(self, g):
        """the start_game event of game g's written log (mjai_log.dump_json_log)"""
        return {"type": "start_game", "names": list(self.names[g]), "seed": [self.seeds[g][0], self.seeds[g][1]]}


def decode_games(games: SelfPlayGames, idx=None, augment: bool = False, device=None):
    """The replay arrays of games idx (default all, in order) -> validate_logs.DecodedLogs with deltas, as decode_dev(<their written
    files>, deltas=True) returns them. Two kernel launches and one copy of the counts to the host. RuntimeError naming the game and
    its seed when its words are corrupt or its log overflowed the arena's capacity."""
    import torch

    from .validate_logs import DecodedLogs

    L = _load()
    idx = list(range(len(games))) if idx is None else [int(i) for i in idx]
    n = len(idx)
    if n == 0:
        raise ValueError("decode_games: no games selected")
    dev = games.words.device if device is None else torch.device("cuda", device)
    if dev.type != "cuda":
        raise ValueError(f"decode_games runs on a CUDA device, got {dev}")
    st = torch.cuda.current_stream(dev).cuda_stream
    sel = torch.tensor(idx, dtype=torch.int64, device=dev)
    words = games.words.to(dev).index_select(0, sel).contiguous()
    lens = games.lens.to(dev).index_select(0, sel).to(torch.int32).contiguous()
    pitch = words.shape[1]
    d_counts = torch.empty((n, 4), dtype=torch.int32, device=dev)
    _lib.check(L.mjx_arena_words_count_dev(n, words.data_ptr(), lens.data_ptr(), pitch, games.log_cap, d_counts.data_ptr(), st),
               "mjx_arena_words_count_dev")
    counts4 = d_counts.cpu().numpy()
    bad = np.nonzero(counts4[:, 0] != STATUS["OK"])[0]
    if len(bad):
        j = int(bad[0])
        g, seed = idx[j], games.seeds[idx[j]]
        if counts4[j, 0] == STATUS["CAPACITY"]:
            why = f"event log overflow: {int(lens[j])} words > capacity {games.log_cap}"
        else:
            why = "corrupt event log: its words are not a sequence of arena events"
        raise RuntimeError(f"self-play game {g} (seed {seed[0]}, {seed[1]}): {why}")
    excl = lambda x: (np.cumsum(x) - x).astype(np.int32)
    ev_cnt, n_ky, n_ho = (counts4[:, k].astype(np.int32) for k in (1, 2, 3))
    ev_off, ky_off, hora_off = excl(ev_cnt), excl(n_ky), excl(n_ho)
    n_ev, n_k, n_h = int(ev_cnt.sum()), int(n_ky.sum()), int(n_ho.sum())
    offs = torch.from_numpy(np.stack([ev_off, ev_cnt, ky_off, hora_off])).to(dev)
    hdr = torch.empty(n_ev, dtype=torch.int64, device=dev)
    lines = torch.empty(n_ev, dtype=torch.int32, device=dev)
    kyoku = torch.empty(n_k * KYOKU_WORDS, dtype=torch.int64, device=dev)
    hora = torch.empty(n_h * HORA_WORDS, dtype=torch.int64, device=dev)
    deltas = torch.empty((n_ev, 4), dtype=torch.int32, device=dev)
    has = torch.zeros(n_ev, dtype=torch.uint8, device=dev)  # the kernel writes the hora and ryukyoku entries only
    ptr = lambda t: t.data_ptr() if t.numel() else None
    _lib.check(L.mjx_arena_words_fill_dev(n, words.data_ptr(), lens.data_ptr(), pitch, games.log_cap, int(augment), d_counts.data_ptr(),
                                          offs[0].data_ptr(), offs[2].data_ptr(), offs[3].data_ptr(), ptr(hdr), ptr(lines), n_ev,
                                          ptr(kyoku), n_k * KYOKU_WORDS, ptr(hora), n_h * HORA_WORDS, ptr(deltas), ptr(has), st),
               "mjx_arena_words_fill_dev")
    # the decoder's counts layout: accept, n_events, n_kyoku, n_hora, then the first line's byte span (no text here: -1)
    counts = np.concatenate([np.ones((n, 1), dtype=np.int32), counts4[:, 1:], np.full((n, 2), -1, dtype=np.int32)], axis=1)
    return DecodedLogs(np.ones(n, dtype=bool), counts, ev_off, ev_cnt, ky_off, hora_off, offs, hdr, lines, kyoku, hora, deltas, has)


class SelfPlayDatasetsIter(FileDatasetsIter):
    """dataloader.FileDatasetsIter whose "files" are the games of a SelfPlayGames: the same arguments with `games` in place of the
    file list. It shuffles a list of game indices of the same length with the same random.shuffle calls, and loads each file batch
    with GameplayLoader.load_games, so for the same state of `random` it yields what FileDatasetsIter yields over the games'
    written files listed in game order."""

    def __init__(self, version, games: SelfPlayGames, pts, oracle=False, file_batch_size=20, reserve_ratio=0, player_names=None,
                 excludes=None, num_epochs=1, enable_augmentation=False, augmented_first=False, *, grp, batch_size, trust_seed=False,
                 device=0):
        super().__init__(version, list(range(len(games))), pts, oracle=oracle, file_batch_size=file_batch_size,
                         reserve_ratio=reserve_ratio, player_names=player_names, excludes=excludes, num_epochs=num_epochs,
                         enable_augmentation=enable_augmentation, augmented_first=augmented_first, grp=grp, batch_size=batch_size,
                         trust_seed=trust_seed, device=device)
        self.games = games

    def _load(self, file_list):
        return self.loader.load_games(self.games, file_list)
