"""libriichi.dataset.GameplayLoader on the CUDA environment (SURVEY.md §8f N3).

Mirror of dataset/gameplay.rs:24-45, 80-218: `GameplayLoader(version, *, oracle, player_names, excludes, trust_seed,
always_include_kan_select, augmented)`, `.load_gz_log_files(filenames) -> list[list[Gameplay]]`, `.load_log(text)`;
`Gameplay.take_obs / take_actions / take_masks / take_at_kyoku / take_dones / take_apply_gamma / take_at_turns /
take_shantens / take_player_id`. The logs are replayed on device (csrc/mjx_replay.cuh) and the observations come from the
same encoder kernels self-play uses. Differences, stated rather than hidden: `take_obs()` / `take_masks()` return ONE tensor
per Gameplay ([n_moves, C, 34] float32 / [n_moves, 46] bool, CUDA by default, `host=True` for numpy) instead of a list of
per-move arrays (`take_invisible_obs()` likewise: [n_moves, 217 | 211, 34]).

With `oracle=False` a log may hide the other seats' tiles, as the mjai protocol shows a game to one seat (their haipai "?" in
start_kyoku, their draws "pai": "?"): as in the reference, only the selected player's own PlayerState is updated, so such a log
loads for the seat that recorded it (select it with `player_names`) to exactly the Gameplays that seat has in the full log. A
player whose own tiles are hidden fails the call with a RuntimeError (mjx error code 13), so the default selection of all four
seats fails on such a log, as it does in the reference. With `oracle=True` every log must carry full information.
With `oracle=True` the hidden tiles come from the game seed when `trust_seed=True` (walls regenerated on device and checked
against the logged deal) and otherwise from the log plus a random fill of the unseen tiles, as dataset/invisible.rs does.
`Grp` (dataset/grp.rs:19-164) is restated in Python (Grp.load_events) and, for whole batches of logs, on the device (k_grp_logs,
csrc/mjx_grp.cuh).

With libmjx built, a CUDA device and a UTF-8 locale, `load_gz_log_files`, `load_logs` and `Grp.load_gz_log_files` decode the log
text on the device (k_mjai_decode with the deltas output, csrc/mjx_mjai.cuh): the event words go to the replay without leaving
the device, and the Grp of every log comes from k_grp_logs. A log the decoder declines, or one that is not UTF-8, is parsed by the
host code below, and so is every log of a batch loaded with `oracle=True, trust_seed=False` (its hidden tiles are drawn from the
caller's numpy `rng`). The results and the exceptions are those of the host code either way.
"""
from __future__ import annotations

import gzip
import json
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import _cdecl, _logio, dataset_codec
from .env import ReplayEnv

_ERR_HIDDEN_OWN_TILE = _cdecl.defines(_cdecl.header())["MJX_REPLAY_ERR_HIDDEN_OWN_TILE"]


class Grp:
    """dataset/grp.rs:19-164: per-kyoku features [grand_kyoku, honba, kyotaku, scores / 10000] (float64 [n_kyoku, 7]),
    the final ranking and final scores of a game. Pure log arithmetic on the host."""

    def __init__(self, feature, rank_by_player, final_scores):
        self.feature, self.rank_by_player, self.final_scores = feature, rank_by_player, final_scores

    @staticmethod
    def load_events(events):
        info, rank, final_deltas, final_scores = [], None, [0, 0, 0, 0], [0, 0, 0, 0]
        for ev in reversed(events):  # grp.rs:96-152 walks the log backwards
            ty = ev["type"]
            if ty in ("hora", "ryukyoku"):
                if rank is None:
                    if ev.get("deltas") is None:
                        raise ValueError("invalid log: field `deltas` is required for Hora and Ryukyoku of AL")
                    final_deltas = [a + b for a, b in zip(final_deltas, ev["deltas"])]
            elif ty == "reach_accepted":
                if rank is None:
                    final_deltas[ev["actor"]] -= 1000
            elif ty == "start_kyoku":
                if rank is None:
                    final_scores = [a + b for a, b in zip(ev["scores"], final_deltas)]
                    order = sorted(range(4), key=lambda i: -final_scores[i])  # rankings.rs:8-22: stable by seat
                    total = sum(final_scores)
                    if total < 100_000:  # leftover riichi sticks go to the top (grp.rs:127-131)
                        final_scores[order[0]] += 100_000 - total
                    rank = [0, 0, 0, 0]
                    for r, pl in enumerate(order):
                        rank[pl] = r
                grand = {"E": ev["kyoku"] - 1, "S": 3 + ev["kyoku"]}.get(ev["bakaze"], 7 + ev["kyoku"])
                info.insert(0, [float(grand), float(ev["honba"]), float(ev["kyotaku"])] + [sc / 10000.0 for sc in ev["scores"]])
        if rank is None:
            raise ValueError("invalid log: no Hora or Ryukyoku after a StartKyoku")
        return Grp(np.array(info, dtype=np.float64).reshape(-1, 7), rank, final_scores)

    @staticmethod
    def load_log(raw_log: str):
        return Grp.load_events(dataset_codec.parse_log(raw_log))

    @staticmethod
    def load_gz_log_files(gzip_filenames):
        """the Grp of every file, in order; on the device (module docstring) when it is ready, in chunks of consecutive files"""
        paths = list(gzip_filenames)
        if paths and _logio.device_ready():
            return _grp_device(paths)
        return [Grp.load_log(_read_gz_text(fn)) for fn in paths]

    def take_feature(self):
        return self.feature

    def take_rank_by_player(self):
        return list(self.rank_by_player)

    def take_final_scores(self):
        return list(self.final_scores)

    def __len__(self):
        return int(self.feature.shape[0])


class Gameplay:
    def __init__(self, player_id: int, player_name: str, obs, actions, masks, at_kyoku, apply_gamma, at_turns, shantens, grp=None,
                 invisible_obs=None):
        self.player_id, self.player_name = player_id, player_name
        self.grp = grp
        self._invisible = invisible_obs
        self._obs, self._masks = obs, masks
        self._actions, self._at_kyoku, self._apply_gamma = actions, at_kyoku, apply_gamma
        self._at_turns, self._shantens = at_turns, shantens
        # gameplay.rs:285-286: done wherever the next move belongs to a later kyoku, and at the last move
        self._dones = np.append(at_kyoku[1:] > at_kyoku[:-1], True) if len(at_kyoku) else np.zeros(0, dtype=bool)

    def take_obs(self, host: bool = False):
        return self._obs.cpu().numpy() if host else self._obs

    def take_masks(self, host: bool = False):
        return self._masks.cpu().numpy() if host else self._masks

    def take_invisible_obs(self, host: bool = False):
        """gameplay.rs:199-201: the invisible (oracle) observation of every move; only with GameplayLoader(oracle=True)"""
        if self._invisible is None:
            raise ValueError("the loader was created with oracle=False")
        return self._invisible.cpu().numpy() if host else self._invisible

    def take_grp(self):
        return self.grp

    def take_actions(self):
        return self._actions.tolist()

    def take_at_kyoku(self):
        return self._at_kyoku.tolist()

    def take_dones(self):
        return self._dones.tolist()

    def take_apply_gamma(self):
        return self._apply_gamma.tolist()

    def take_at_turns(self):
        return self._at_turns.tolist()

    def take_shantens(self):
        return self._shantens.tolist()

    def take_player_id(self):
        return self.player_id


class GameplayLoader:
    def __init__(self, version: int, *, oracle: bool = True, player_names=None, excludes=None, trust_seed: bool = False,
                 always_include_kan_select: bool = True, augmented: bool = False, device: int = 0, shuffle_kind: int = 0, rng=None):
        # gameplay.rs:80-113: same keywords and defaults (oracle = true, always_include_kan_select = true); `shuffle_kind` selects the
        # wall shuffle of the seeds (see mjx_env_create), `rng` the numpy Generator behind the random fill of unseen tiles
        if oracle and trust_seed and augmented:
            raise NotImplementedError("oracle + trust_seed + augmented: the regenerated walls would not match the augmented events "
                                      "(the reference mismatches them too, dataset/invisible.rs:51-66)")
        self.version, self.oracle, self.trust_seed = version, oracle, trust_seed
        self.shuffle_kind = shuffle_kind
        self.rng = rng if rng is not None else np.random.default_rng()
        self.player_names, self.excludes = list(player_names or []), list(excludes or [])
        self.always_include_kan_select, self.augmented = always_include_kan_select, augmented
        self.device = device

    def _players(self, names):  # gameplay.rs:166-176
        if self.player_names:
            return [i for i, nm in enumerate(names) if nm in set(self.player_names)]
        if self.excludes:
            return [i for i, nm in enumerate(names) if nm not in set(self.excludes)]
        return [0, 1, 2, 3]

    def load_log(self, raw_log: str):
        return self.load_logs([raw_log])[0]

    def _on_device(self) -> bool:
        # oracle=True, trust_seed=False: reconstruct_walls draws every kyoku's unseen tiles from self.rng on the host
        return not (self.oracle and not self.trust_seed) and _logio.device_ready()

    def load_gz_log_files(self, gzip_filenames):
        if not self._on_device():
            texts = []
            for fn in gzip_filenames:
                texts.append(_read_gz_text(fn))
            return self._load_host(texts)
        paths = list(gzip_filenames)
        with ThreadPoolExecutor(max(1, min(32, os.cpu_count() or 1, len(paths)))) as pool:  # zlib and file reads release the GIL
            blobs = list(pool.map(_logio.read_gz, paths))
        logs = []
        for fn, b in zip(paths, blobs):
            if b is None or not _logio.utf8_ok(b):  # the host reader raises its own exception (or reads the file after all)
                logs.append(_Log(text=_read_gz_text(fn)))
            else:
                logs.append(_Log(blob=b))
        return self._load_device(logs)

    def load_logs(self, texts):
        """list of log texts -> list (per log) of list (per selected player) of Gameplay; all logs replayed as one batch"""
        if not self._on_device():
            return self._load_host(texts)
        logs = []
        for t in texts:
            try:
                logs.append(_Log(text=t, blob=t.encode("utf-8")))
            except UnicodeEncodeError:  # lone surrogates: not UTF-8, so the host decides
                logs.append(_Log(text=t))
        return self._load_device(logs)

    def _load_host(self, texts):
        """load_logs with every log parsed, encoded and scored on the host"""
        games = [dataset_codec.parse_log(t) for t in texts]
        if self.augmented:  # gameplay.rs:126-128: manzu <-> pinzu on every event before anything else
            games = [dataset_codec.augment_events(ev) for ev in games]
        for ev in games:
            if not ev or ev[0].get("type") != "start_game" or len(ev) < 4:
                raise ValueError("empty or invalid game log")
        players = [self._players(ev[0].get("names", ["", "", "", ""])) for ev in games]
        walls = None
        if self.oracle and not self.trust_seed:  # dataset/invisible.rs:24-148: from the log, unseen tiles filled at random
            walls = [dataset_codec.reconstruct_walls(ev, self.rng) for ev in games]
        jobs = dataset_codec.build_jobs(games, players, walls)
        return self._replay(jobs, [ev[0] for ev in games], lambda: [Grp.load_events(ev) for ev in games])

    def _load_device(self, logs):
        """load_logs over _Log items: decoded on the device (module docstring), the rest through the host code; the checks and
        exceptions come in the host path's order"""
        import torch

        from . import _lib
        from .validate_logs import decode_dev

        n = len(logs)
        dev_idx = [k for k, lg in enumerate(logs) if lg.blob is not None]
        slot = {k: j for j, k in enumerate(dev_idx)}
        D = G = None
        with torch.cuda.device(self.device):
            _lib.init(self.device)
            if dev_idx:
                D = decode_dev([logs[k].blob for k in dev_idx], self.device, augment=self.augmented, deltas=True)
                G = _grp_run(D, self.device, with_types=self.augmented)
        host = [k for k in range(n) if k not in slot or not D.accept[slot[k]] or
                (self.augmented and not _augment_safe(logs[k].blob, G.types[slot[k]]))]
        on_host = set(host)
        games = {k: dataset_codec.parse_log(logs[k].host_text()) for k in host}  # parse errors first, in log order
        if self.augmented:
            games = {k: dataset_codec.augment_events(games[k]) for k in host}
        for k in range(n):
            if k in on_host:
                ev = games[k]
                if not ev or ev[0].get("type") != "start_game" or len(ev) < 4:
                    raise ValueError("empty or invalid game log")
            elif G.first_type[slot[k]] != dataset_codec.START_GAME or D.ev_cnt[slot[k]] < 4:
                raise ValueError("empty or invalid game log")
        firsts = []
        for k in range(n):  # the first event: names and seed (the decoder reports its line as a byte span)
            if k in on_host:
                firsts.append(games[k][0])
            else:
                b, e = (int(x) for x in D.counts[slot[k], 4:6])
                firsts.append(json.loads(logs[k].blob[b:e].decode("utf-8")))
        players = [self._players(f.get("names", ["", "", "", ""])) for f in firsts]
        # the jobs: the decoded arrays on the device, the host-encoded logs' words and payloads appended after them
        dev = torch.device("cuda", self.device)
        hdr = [D.hdr] if D is not None else []
        kyoku = [D.kyoku] if D is not None else []
        nh = D.hdr.numel() if D is not None else 0
        nk = D.kyoku.numel() // dataset_codec.KYOKU_WORDS if D is not None else 0
        ev_off, ev_cnt, ky_off, pids, job_game = [], [], [], [], []
        for g in range(n):
            if g in on_host:
                h, p = dataset_codec.encode_events(games[g])
                span = (nh, len(h), nk)
                hdr.append(torch.from_numpy(h.view(np.int64)).to(dev)); kyoku.append(torch.from_numpy(p.reshape(-1).view(np.int64)).to(dev))
                nh += len(h); nk += len(p)
            else:
                j = slot[g]
                span = (int(D.ev_off[j]), int(D.ev_cnt[j]), int(D.ky_off[j]))
            for pid in players[g]:
                ev_off.append(span[0]); ev_cnt.append(span[1]); ky_off.append(span[2]); pids.append(pid); job_game.append(g)
        cat = lambda xs: torch.cat(xs) if xs else torch.zeros(0, dtype=torch.int64, device=dev)
        jobs = dict(hdr=cat(hdr), kyoku=cat(kyoku), ev_off=np.array(ev_off, dtype=np.int32), ev_cnt=np.array(ev_cnt, dtype=np.int32),
                    ky_off=np.array(ky_off, dtype=np.int32), players=np.array(pids, dtype=np.uint8),
                    job_game=np.array(job_game, dtype=np.int32))

        def grps():
            out = []
            for g in range(n):
                if g in on_host:
                    out.append(Grp.load_events(games[g]))
                    continue
                grp = G.grp(D, slot[g])
                if grp is None:  # k_grp_logs declined: the host raises its exception for this log
                    ev = dataset_codec.parse_log(logs[g].host_text())
                    grp = Grp.load_events(dataset_codec.augment_events(ev) if self.augmented else ev)
                out.append(grp)
            return out

        return self._replay(jobs, firsts, grps)

    def _replay(self, jobs, firsts, grps):
        """the replay of the jobs -> load_logs's result; firsts = every log's first event, grps() = every log's Grp"""
        import torch

        n_jobs = len(jobs["players"])
        out = [[] for _ in firsts]
        if n_jobs == 0:
            return out
        env = ReplayEnv(jobs, obs_version=self.version, always_include_kan_select=self.always_include_kan_select, device=self.device)
        chunks = []  # per step: (job ids, obs, masks, labels, meta[, invisible obs])
        try:
            if self.oracle and self.trust_seed:  # invisible.rs:35-66: the walls are those of the game's seed
                seeds = []
                for first in firsts:
                    sd = first.get("seed")
                    if sd is None:
                        raise ValueError("trust_seed=True needs start_game.seed in every log")
                    seeds.append((int(sd[0]), int(sd[1])))
                env.trust_seeds([seeds[g][0] for g in jobs["job_game"]], [seeds[g][1] for g in jobs["job_game"]], self.shuffle_kind)
            elif not self.oracle:  # gameplay.rs:240-335: only the player's own PlayerState is updated, so other seats may be `?`
                env.viewpoints()
            while True:
                env.replay_step()
                nr = env.num_rows()
                if nr:
                    obs = env.encode_obs()[:nr]
                    chunk = (env.row_table[:nr].long().clone(), obs.clone(), env.masks[:nr].clone(),
                             env.row_label[:nr].clone(), env.row_meta[:nr].clone())
                    if self.oracle:
                        chunk += (env.encode_invisible(self.version)[:nr].clone(),)
                    chunks.append(chunk)
                if env.num_live() == 0:
                    break
            res = env.results()
            sp_overflows = env.sp_overflows() if self.version == 4 else 0
        finally:
            env.close()
        if sp_overflows:
            raise RuntimeError(f"single-player state arena overflowed in {sp_overflows} replay step(s): observation rows 889-1011 "
                               "would be zero; load fewer logs per call")
        if (res["err"] != 0).any():
            bad = int(np.nonzero(res["err"])[0][0])
            code = int(res["err"][bad])
            why = ("the player's own tiles are hidden in this log (attempt to witness an unknown tile); a log recorded from one "
                   "seat loads for that seat only, selected with player_names" if code == _ERR_HIDDEN_OWN_TILE
                   else "the log is inconsistent or not full-information")
            raise RuntimeError(f"replay job {bad} (log {int(jobs['job_game'][bad])}, player {int(jobs['players'][bad])}) failed "
                               f"with mjx error code {code}: {why}")
        if chunks:
            job = torch.cat([c[0] for c in chunks]); obs = torch.cat([c[1] for c in chunks]); masks = torch.cat([c[2] for c in chunks])
            label = torch.cat([c[3] for c in chunks]); meta = torch.cat([c[4] for c in chunks])
            order = torch.sort(job, stable=True).indices  # moves of a job stay in emission order
            inv = torch.cat([c[5] for c in chunks])[order] if self.oracle else None
            job, obs, masks, label, meta = job[order], obs[order], masks[order], label[order].cpu().numpy(), meta[order].cpu().numpy()
            counts = torch.bincount(job, minlength=n_jobs).cpu().numpy()
        else:
            counts = np.zeros(n_jobs, dtype=np.int64)
        grps = grps()
        start = 0
        for j in range(n_jobs):
            n = int(counts[j]); sl = slice(start, start + n); start += n
            g, pid = int(jobs["job_game"][j]), int(jobs["players"][j])
            name = firsts[g].get("names", ["", "", "", ""])[pid]
            if n:
                gp = Gameplay(pid, name, obs[sl], label[sl], masks[sl], meta[sl, 0].copy(), meta[sl, 3].astype(bool),
                              meta[sl, 1].copy(), meta[sl, 2].astype(np.int8), grp=grps[g], invisible_obs=None if inv is None else inv[sl])
            else:
                z = np.zeros(0, dtype=np.uint8)
                gp = Gameplay(pid, name, torch.zeros((0, env.obs_rows, 34), device=obs.device if chunks else "cpu"), np.zeros(0, dtype=np.int64),
                              torch.zeros((0, 46), dtype=torch.bool), z, z.astype(bool), z, z.astype(np.int8), grp=grps[g])
            out[g].append(gp)
        return out


def _read_gz_text(fn):
    """the host reader of a log file: gunzip, the locale's encoding, universal newlines"""
    with gzip.open(fn, "rt") as f:
        return f.read()


class _Log:
    """one log of a device load: `blob` = its UTF-8 bytes for the decoder (None: the host parses it), `text` = the str the host
    code parses (made from the blob as the host reader would, when needed)"""

    def __init__(self, text=None, blob=None):
        self.text, self.blob = text, blob

    def host_text(self):
        if self.text is None:
            self.text = _logio.host_text(self.blob)
        return self.text


# augment_events swaps the tiles of these fields on every event that has them; the decoder validates a field only for the event
# types that read it (the MJT_* codes), so a log with the field anywhere else goes to the host, whose augment_events decides
_AUGMENTED_FIELDS = (
    (b'"pai"', (dataset_codec.TSUMO, dataset_codec.DAHAI, dataset_codec.CHI, dataset_codec.PON, dataset_codec.DAIMINKAN,
                dataset_codec.KAKAN)),
    (b'"dora_marker"', (dataset_codec.START_KYOKU, dataset_codec.DORA)),
    (b'"bakaze"', (dataset_codec.START_KYOKU,)),
    (b'"consumed"', (dataset_codec.CHI, dataset_codec.PON, dataset_codec.DAIMINKAN, dataset_codec.KAKAN, dataset_codec.ANKAN)),
    (b'"tehais"', (dataset_codec.START_KYOKU,)),
    (b'"ura_markers"', (dataset_codec.HORA,)),
)


def _augment_safe(blob: bytes, types) -> bool:
    """whether every field augment_events rewrites sits on an event whose type the decoder checked it for: a key is never escaped
    in an accepted log, so it appears in the text at least once per event that has it (more often only inside other strings
    or values, which merely sends the log to the host); `types` = the log's event count per type"""
    return all(blob.count(key) <= sum(int(types[t]) for t in ts) for key, ts in _AUGMENTED_FIELDS)


class _GrpRun:
    """k_grp_logs over a DecodedLogs, copied back once: status, ranks, final scores and feature rows per log, plus the type of
    every log's first event and (with_types) its event count per type"""

    def __init__(self, flat, n, n_rows, with_types):
        sizes = [n, 4 * n, 4 * n, 7 * n_rows, n] + ([17 * n] if with_types else [])
        parts = np.split(flat, np.cumsum(sizes)[:-1])
        self.status, self.first_type = parts[0], parts[4]
        self.rank, self.final, self.feat = parts[1].reshape(n, 4), parts[2].reshape(n, 4), parts[3].reshape(n_rows, 7)
        self.types = parts[5].reshape(n, 17) if with_types else None

    def grp(self, D, j):
        """the Grp of log j, or None when its status is not OK"""
        if self.status[j] != 0:
            return None
        lo = int(D.ky_off[j])
        feature = self.feat[lo:lo + int(D.counts[j, 2])].astype(np.float64)
        feature[:, 3:] /= 10000.0
        return Grp(feature, self.rank[j].tolist(), self.final[j].tolist())


def _grp_run(D, device: int, with_types: bool = False) -> _GrpRun:
    """mjx_grp_logs_dev over decode_dev(..., deltas=True)'s arrays and one copy back (_GrpRun)"""
    import torch

    from . import _lib

    L = _lib.load()
    dev = torch.device("cuda", device)
    n = len(D.accept)
    n_rows = D.kyoku.numel() // dataset_codec.KYOKU_WORDS
    feat = torch.empty((n_rows, 7), dtype=torch.int32, device=dev)
    rank = torch.empty((n, 4), dtype=torch.uint8, device=dev)
    final = torch.empty((n, 4), dtype=torch.int64, device=dev)
    status = torch.empty(n, dtype=torch.int32, device=dev)
    ptr = lambda t: t.data_ptr() if t.numel() else None
    _lib.check(L.mjx_grp_logs_dev(n, ptr(D.hdr), D.offs[0].data_ptr(), D.offs[1].data_ptr(), D.hdr.numel(), ptr(D.kyoku),
                                  D.offs[2].data_ptr(), D.kyoku.numel(), ptr(D.deltas), ptr(D.has_deltas), ptr(feat), rank.data_ptr(),
                                  final.data_ptr(), status.data_ptr(), torch.cuda.current_stream(dev).cuda_stream), "mjx_grp_logs_dev")
    first = torch.full((n,), -1, dtype=torch.int64, device=dev)
    acc = torch.from_numpy(np.nonzero(D.ev_cnt > 0)[0]).to(dev)
    if acc.numel():
        first[acc] = D.hdr[D.offs[0][acc].long()] & 0xFF
    parts = [status.long(), rank.long().flatten(), final.flatten(), feat.long().flatten(), first]
    if with_types:  # the event count per type of every log
        log_of = torch.repeat_interleave(torch.arange(n, device=dev), D.offs[1].long(), output_size=D.hdr.numel())
        parts.append(torch.bincount(log_of * 17 + (D.hdr & 0xFF), minlength=17 * n))
    return _GrpRun(torch.cat(parts).cpu().numpy(), n, n_rows, with_types)


def _grp_device(paths):
    """Grp.load_gz_log_files on the device (_logio.log_device()): per chunk of files, read + gunzip on a thread pool, decode with
    the deltas output, k_grp_logs, one copy back; the files it cannot take, in order, through the host code"""
    import torch

    from . import _lib
    from .validate_logs import decode_dev

    device = _logio.log_device()
    _lib.init(device)
    out = []
    workers = min(32, os.cpu_count() or 1)
    # torch.cuda.device: the streams and allocations below belong to `device` whatever torch's current device is
    with torch.cuda.device(device), ThreadPoolExecutor(workers) as pool:  # zlib and file reads release the GIL
        for chunk, blobs in _logio.chunks(paths, pool, 4 * workers, _logio.read_gz, _logio.CHUNK_LOGS, _logio.CHUNK_BYTES):
            res = [None] * len(chunk)
            on_dev = [k for k, b in enumerate(blobs) if b is not None]  # a file that is not UTF-8 is declined by the decoder
            if on_dev:
                D = decode_dev([blobs[k] for k in on_dev], device, deltas=True)
                G = _grp_run(D, device)
                for j, k in enumerate(on_dev):
                    if D.accept[j]:
                        res[k] = G.grp(D, j)
            for k, path in enumerate(chunk):
                if res[k] is None:
                    res[k] = Grp.load_log(_read_gz_text(path))
            out += res
    return out
