"""mortal/one_vs_three.py on the device: `python -m mortal_b200.one_vs_three [CONFIG] [--summary PATH]`, or
`one_vs_three(config, iters=None, out=None)` (out: sys.stdout).

It reads the `[1v3]` section of the reference's config.toml (the file named on the command line, else $MORTAL_CFG, else
./config.toml) and plays the challenger checkpoint against the champion checkpoint in 1v3 duplicate games: every seed four times,
with the challenger at each seat once (libriichi.arena.OneVsThree.py_vs_py). Iteration i plays `games_per_iter // 4` seeds from
10000 + i * (games_per_iter // 4) on with the run's `seed_key` (-1 or absent: a random 64-bit key, logged so the run can be
repeated), and prints the reference's three lines for it:

    --------------------------------------------------
    # 0
    challenger rankings: [503 498 501 498] (2.4975, 1.035pt)

Both engines are `DeviceEngine`s over `model.load_mortal` of the sections' `state_file`, with their `name`, `enable_amp`,
`enable_rule_based_agari_guard` and `stochastic_latent`; `enable_compile` is read and not applied. With a non-empty `log_dir` the
games' logs are written there as py_vs_py writes them (`{seed}_{key}_{a|b|c|d}.json.gz`); absent or '' writes nothing.

Beyond the reference:
- Every game is recorded on the device (`record_games`) and both sides' statistics are taken from the words
  (`stat.Stat.from_games`), so no log has to be written or read back for them. After the last iteration a report follows the
  iteration lines: each side's `Stat` report (what `python -m mortal_b200.stat LOG_DIR NAME` prints over the run's logs) under
  a header naming it and its seats per game, then the challenger's average rank pt with its standard error over duplicate sets
  (a set is the four games of one seed; the per-set mean is the independent unit). `--summary PATH` writes the same as JSON.
- `[1v3] iters_per_call` (default 1, one arena per iteration as in the reference) plays that many iterations' seeds in one
  py_vs_py call, a larger batch for the GPU; the rankings of each iteration are split from the call's rank rows by seed. The
  output lines and the log file names are the same. The games are the same too for engines whose actions do not depend on the
  batch they are evaluated in; a network's bf16 forward may round differently at another batch size.
- An oracle checkpoint plays as an oracle engine: the arena hands it the invisible observation. The reference builds every
  engine with is_oracle=False and cannot run one.
- Rejected before any model is loaded: `[1v3.akochan] enabled = true` (NotImplementedError, akochan agents are not supported),
  fewer than 4 games per iteration, a challenger and champion on different devices or not on a CUDA device (the arena plays both
  engines on one GPU), and a challenger and champion with the same name (their statistics could not be told apart).
"""
from __future__ import annotations

import argparse
import json
import logging
import math
import secrets
import sys
from dataclasses import dataclass

import numpy as np

from .libriichi.arena import AKOCHAN_UNSUPPORTED, OneVsThree
from .stat import COUNTERS, Stat

PTS = [90, 45, 0, -135]
SEED_START = 10000  # one_vs_three.py: seed_start


@dataclass
class Plan:
    """the [1v3] section, checked and resolved"""
    key: int               # the seed key of every game
    key_drawn: bool        # seed_key was -1 or absent: key was drawn with secrets.randbits(64)
    seeds_per_iter: int
    seeds: list            # the first seed of every iteration (the reference's range)
    iters_per_call: int
    log_dir: str | None
    device: int            # the CUDA device index of both engines and the arena


def plan(config, iters=None) -> Plan:
    """config['1v3'] checked and resolved, before anything is loaded; `iters` overrides [1v3] iters"""
    import torch

    cfg = config["1v3"]
    if cfg.get("akochan", {}).get("enabled", False):
        raise NotImplementedError(AKOCHAN_UNSUPPORTED)
    seeds_per_iter = int(cfg["games_per_iter"]) // 4
    if seeds_per_iter < 1:
        raise ValueError(f"[1v3] games_per_iter = {cfg['games_per_iter']} gives 0 seeds per iteration (games_per_iter // 4)")
    iters = int(cfg["iters"] if iters is None else iters)
    if iters < 0:
        raise ValueError(f"[1v3] iters = {iters} is negative")
    iters_per_call = cfg.get("iters_per_call", 1)
    if not isinstance(iters_per_call, int) or iters_per_call < 1:
        raise ValueError(f"[1v3] iters_per_call = {iters_per_call!r}: a positive integer expected")
    chal, cham = cfg["challenger"], cfg["champion"]
    devs = []
    for side, sec in (("challenger", chal), ("champion", cham)):
        d = torch.device(sec["device"])
        if d.type != "cuda":
            raise ValueError(f"[1v3.{side}] device = {sec['device']!r}: the arena plays on a CUDA device")
        devs.append(0 if d.index is None else d.index)
    if devs[0] != devs[1]:
        raise ValueError(f"[1v3] challenger device {chal['device']!r} and champion device {cham['device']!r} differ: the arena "
                         "plays both engines on one GPU")
    if str(chal["name"]) == str(cham["name"]):
        raise ValueError(f"[1v3] challenger and champion are both named {chal['name']!r}: their statistics could not be told apart")
    key = cfg.get("seed_key", -1)
    drawn = key == -1
    if drawn:
        key = secrets.randbits(64)
    seeds = list(range(SEED_START, SEED_START + seeds_per_iter * iters, seeds_per_iter))
    return Plan(int(key), drawn, seeds_per_iter, seeds, iters_per_call, cfg.get("log_dir") or None, devs[0])


def load_engine(section, device: int):
    """a DeviceEngine over the checkpoint of a [1v3.challenger] / [1v3.champion] section"""
    import torch

    from .engine import DeviceEngine
    from .model import load_mortal

    state = torch.load(section["state_file"], weights_only=True, map_location="cpu")
    brain, dqn = load_mortal(state)
    _ = section.get("enable_compile", False)  # read, not applied (module docstring)
    return DeviceEngine(brain, dqn, version=brain.version, device=torch.device("cuda", device), enable_amp=section["enable_amp"],
                        enable_rule_based_agari_guard=section["enable_rule_based_agari_guard"], name=section["name"],
                        is_oracle=brain.is_oracle, stochastic_latent=section.get("stochastic_latent", False))


@dataclass
class Result:
    key: int
    seeds_per_iter: int
    seeds: list               # the first seed of every iteration; iteration i plays seeds[i] .. seeds[i] + seeds_per_iter - 1
    rankings: np.ndarray      # int64 [iters, 4]: the challenger's 1st..4th places per iteration
    set_pts: np.ndarray       # float64 [iters * seeds_per_iter]: the challenger's mean rank pt over the four games of each seed
    names: tuple              # (challenger, champion)
    challenger: Stat
    champion: Stat

    @property
    def avg_pt(self) -> float:
        return float(self.set_pts.mean()) if len(self.set_pts) else math.nan

    @property
    def avg_pt_stderr(self) -> float:
        n = len(self.set_pts)
        return float(self.set_pts.std(ddof=1) / math.sqrt(n)) if n > 1 else math.nan

    def report(self) -> str:
        """both sides' Stat reports, then the challenger's average rank pt with its standard error over duplicate sets"""
        blocks = [f"{role} {name} (x{seats})\n{st.reference_text()}"
                  for role, name, seats, st in (("challenger", self.names[0], 1, self.challenger),
                                                ("champion", self.names[1], 3, self.champion))]
        blocks.append(f"challenger avg rank pt {self.avg_pt:.6f} ± {self.avg_pt_stderr:.6f} "
                      f"(standard error over {len(self.set_pts)} duplicate sets of 4 games)")
        return "=" * 50 + "\n" + "\n\n".join(blocks)

    def summary(self) -> dict:
        finite = lambda x: x if math.isfinite(x) else None
        side = lambda name, seats, st: {"name": name, "seats": seats, "counters": {c: getattr(st, c) for c in COUNTERS}}
        return {"seed_key": self.key, "seeds_per_iter": self.seeds_per_iter, "seeds": list(self.seeds),
                "rankings": self.rankings.tolist(), "avg_pt": finite(self.avg_pt), "avg_pt_stderr": finite(self.avg_pt_stderr),
                "challenger": side(self.names[0], 1, self.challenger), "champion": side(self.names[1], 3, self.champion)}


def _print_rankings(rankings, out):
    """the reference's rankings line of an iteration, with its numpy expressions"""
    avg_rank = rankings @ np.arange(1, 5) / rankings.sum()
    avg_pt = rankings @ np.array([90, 45, 0, -135]) / rankings.sum()
    print(f'challenger rankings: {rankings} ({avg_rank}, {avg_pt}pt)', file=out)


def one_vs_three(config, iters=None, out=None) -> Result:
    """mortal/one_vs_three.py main() over `config` (the whole config.toml as a dict), printing to `out` (default: sys.stdout at
    the time of the call); `iters` overrides [1v3] iters. Returns the Result: per-iteration rankings, seeds, both sides'
    accumulated Stat."""
    out = sys.stdout if out is None else out
    P = plan(config, iters)
    cfg = config["1v3"]
    if P.key_drawn:
        logging.info(f"seed_key {P.key} (drawn; set [1v3] seed_key = {P.key} to repeat this run)")
    names = (str(cfg["challenger"]["name"]), str(cfg["champion"]["name"]))
    chal = load_engine(cfg["challenger"], P.device)
    cham = load_engine(cfg["champion"], P.device)
    spi, n_iter = P.seeds_per_iter, len(P.seeds)
    rankings = np.zeros((n_iter, 4), dtype=np.int64)
    set_pts = np.zeros(n_iter * spi, dtype=np.float64)
    st_chal, st_cham = Stat(), Stat()
    pts = np.array(PTS, dtype=np.float64)
    for c0 in range(0, n_iter, P.iters_per_call):
        m = min(P.iters_per_call, n_iter - c0)
        print('-' * 50, file=out)
        print('#', c0, file=out)
        out.flush()
        arena = OneVsThree(disable_progress_bar=False, log_dir=P.log_dir, device=P.device)
        arena.record_games = True
        arena.py_vs_py(challenger=chal, champion=cham, seed_start=(P.seeds[c0], P.key), seed_count=m * spi)
        ranks = arena.last_results["ranks"]
        g = np.arange(ranks.shape[0])
        chal_rank = ranks[g, g % 4].astype(np.int64)  # game 4 * s + r: the challenger sits at seat r (one_vs_three.rs:55-60)
        rankings[c0:c0 + m] = (chal_rank.reshape(m, 4 * spi, 1) == np.arange(4)).sum(1)
        set_pts[c0 * spi:(c0 + m) * spi] = pts[chal_rank].reshape(m * spi, 4).mean(1)
        games, arena.last_games = arena.last_games, None
        st_chal = st_chal + Stat.from_games(games, names[0])
        st_cham = st_cham + Stat.from_games(games, names[1])
        del games, arena  # the words are freed before the next call plays
        for i in range(c0, c0 + m):
            if i > c0:
                print('-' * 50, file=out)
                print('#', i, file=out)
            _print_rankings(rankings[i], out)
        out.flush()
    result = Result(P.key, spi, P.seeds, rankings, set_pts, names, st_chal, st_cham)
    print(result.report(), file=out)
    return result


def main(argv=None) -> int:
    from .train_grp import load_config

    ap = argparse.ArgumentParser(prog="python -m mortal_b200.one_vs_three",
                                 description="Play a challenger checkpoint against a champion in 1v3 duplicate games ([1v3]).")
    ap.add_argument("config", nargs="?", help="config.toml (default: $MORTAL_CFG, else ./config.toml)")
    ap.add_argument("--summary", metavar="PATH", help="also write the seeds, rankings and both sides' counters as JSON")
    args = ap.parse_args(sys.argv[1:] if argv is None else argv)
    logging.basicConfig(level=logging.INFO, format="%(asctime)s %(levelname)s %(message)s")
    try:
        result = one_vs_three(load_config(args.config))
    except KeyboardInterrupt:
        return 0
    if args.summary:
        with open(args.summary, "w") as f:
            json.dump(result.summary(), f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
