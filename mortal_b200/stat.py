"""libriichi.stat.Stat — per-player statistics over mjai logs (stat.rs:26-124 fields, 263-442 accumulation, 447-515 loaders,
516-786 derived rates); used by mortal/player.py:71 and the test-play report of mortal/train.py:321-350. Counters are plain
integer attributes with the reference's names; every derived quantity is a property `numerator / denominator` in float64 with
IEEE semantics (0/0 = nan, x/0 = ±inf) like the Rust `as f64` divisions.

    Stat.from_dir(dir, player_name)            (every dir/**/*.json and dir/**/*.json.gz)
    python -m mortal_b200.stat DIR PLAYER_NAME (bin/stat.rs: prints the reference's report)

With libmjx built and a CUDA device present, from_dir decodes the log texts on the device (k_mjai_decode with the deltas output,
csrc/mjx_mjai.cuh) and runs Stat.from_game there for every selected seat (k_stat_logs, csrc/mjx_stat.cuh); the counters are
summed on the device and copied back once per chunk. A file the device cannot take as it is (unreadable, not gzip, not UTF-8,
declined by the decoder, a hora or ryukyoku without deltas for a selected seat, a first event that is not start_game, a selected
seat past 3) is read by the host code below, so it gives the same counters or raises the same exception. Without the library or
a device, every file is read on the host.
"""
from __future__ import annotations

import glob
import gzip
import json
import math
import os
import sys
from concurrent.futures import ThreadPoolExecutor

from . import _logio
from ._logio import device_ready as _device_ready, log_device as _stat_device, read_bytes as _read_bytes  # noqa: F401

COUNTERS = (
    "game round oya point rank_1 rank_2 rank_3 rank_4 tobi "
    "agari agari_as_oya agari_jun agari_point_oya agari_point_ko "
    "riichi riichi_as_oya riichi_jun chasing_riichi riichi_got_chased riichi_agari riichi_agari_jun riichi_agari_point "
    "riichi_houjuu riichi_ryukyoku riichi_point "
    "fuuro fuuro_num fuuro_agari fuuro_agari_jun fuuro_agari_point fuuro_houjuu fuuro_point "
    "dama_agari dama_agari_jun dama_agari_point "
    "houjuu houjuu_jun houjuu_to_oya houjuu_point_to_oya houjuu_point_to_ko "
    "ryukyoku ryukyoku_point yakuman nagashi_mangan"
).split()

# derived quantity -> (numerator expression, denominator expression) over the counters (stat.rs:555-786)
RATES = {
    "rank_1_rate": ("rank_1", "game"), "rank_2_rate": ("rank_2", "game"), "rank_3_rate": ("rank_3", "game"),
    "rank_4_rate": ("rank_4", "game"), "tobi_rate": ("tobi", "game"),
    "avg_point_per_game": ("point", "game"), "avg_point_per_round": ("point", "round"),
    "avg_point_per_agari": ("agari_point_ko + agari_point_oya", "agari"),
    "avg_point_per_oya_agari": ("agari_point_oya", "agari_as_oya"),
    "avg_point_per_ko_agari": ("agari_point_ko", "agari - agari_as_oya"),
    "avg_point_per_riichi_agari": ("riichi_agari_point", "riichi_agari"),
    "avg_point_per_fuuro_agari": ("fuuro_agari_point", "fuuro_agari"),
    "avg_point_per_dama_agari": ("dama_agari_point", "dama_agari"),
    "avg_point_per_ryukyoku": ("ryukyoku_point", "ryukyoku"),
    "avg_agari_jun": ("agari_jun", "agari"), "avg_riichi_agari_jun": ("riichi_agari_jun", "riichi_agari"),
    "avg_fuuro_agari_jun": ("fuuro_agari_jun", "fuuro_agari"), "avg_dama_agari_jun": ("dama_agari_jun", "dama_agari"),
    "avg_point_per_houjuu": ("houjuu_point_to_ko + houjuu_point_to_oya", "houjuu"),
    "avg_point_per_houjuu_to_oya": ("houjuu_point_to_oya", "houjuu_to_oya"),
    "avg_point_per_houjuu_to_ko": ("houjuu_point_to_ko", "houjuu - houjuu_to_oya"),
    "avg_houjuu_jun": ("houjuu_jun", "houjuu"),
    "agari_rate": ("agari", "round"), "houjuu_rate": ("houjuu", "round"), "riichi_rate": ("riichi", "round"),
    "fuuro_rate": ("fuuro", "round"), "ryukyoku_rate": ("ryukyoku", "round"),
    "agari_rate_after_riichi": ("riichi_agari", "riichi"), "houjuu_rate_after_riichi": ("riichi_houjuu", "riichi"),
    "chasing_riichi_rate": ("chasing_riichi", "riichi"), "riichi_chased_rate": ("riichi_got_chased", "riichi"),
    "avg_riichi_jun": ("riichi_jun", "riichi"), "avg_riichi_point": ("riichi_point", "riichi"),
    "agari_rate_as_oya": ("agari_as_oya", "oya"), "agari_as_oya_rate": ("agari_as_oya", "agari"),
    "houjuu_to_oya_rate": ("houjuu_to_oya", "houjuu"),
    "avg_fuuro_num": ("fuuro_num", "fuuro"), "agari_rate_after_fuuro": ("fuuro_agari", "fuuro"),
    "houjuu_rate_after_fuuro": ("fuuro_houjuu", "fuuro"), "avg_fuuro_point": ("fuuro_point", "fuuro"),
    "yakuman_rate": ("yakuman", "round"), "nagashi_mangan_rate": ("nagashi_mangan", "round"),
}
# from_dir's device path decodes and counts the files in chunks of consecutive files: at most CHUNK_LOGS files and, unless a
# single file is larger, CHUNK_BYTES of decompressed text (_logio.py).
CHUNK_LOGS = _logio.CHUNK_LOGS
CHUNK_BYTES = _logio.CHUNK_BYTES


def _fdiv(a: float, b: float) -> float:
    if b == 0:
        return float("nan") if a == 0 else (float("inf") if a > 0 else float("-inf"))
    return a / b


class Stat:
    def __init__(self, **counters):
        for name in COUNTERS:
            setattr(self, name, int(counters.get(name, 0)))

    def __getattr__(self, name):  # derived rates (only reached for names that are not counters)
        spec = RATES.get(name)
        if spec is None:
            raise AttributeError(name)
        env = {c: getattr(self, c) for c in COUNTERS}
        return _fdiv(float(eval(spec[0], {}, env)), float(eval(spec[1], {}, env)))

    def __add__(self, other: "Stat") -> "Stat":  # stat.rs Sum / Add: field-wise
        return Stat(**{c: getattr(self, c) + getattr(other, c) for c in COUNTERS})

    def __radd__(self, other):
        return self if other == 0 else self.__add__(other)

    def total_pt(self, pts) -> int:
        return self.rank_1 * pts[0] + self.rank_2 * pts[1] + self.rank_3 * pts[2] + self.rank_4 * pts[3]

    def avg_pt(self, pts) -> float:
        return _fdiv(float(self.total_pt(pts)), float(self.game))

    @property
    def avg_rank(self) -> float:
        return self.avg_pt([1, 2, 3, 4])

    # ---------------------------------------------------------------- stat.rs:263-442
    @staticmethod
    def from_game(events, player_id: int) -> "Stat":
        st = Stat(game=1)
        me = player_id
        scores = [0, 0, 0, 0]
        declared = accepted = others_declared = False
        oya = jun = calls = 0
        for ev in events:
            ty = ev["type"]
            if ty == "start_kyoku":
                st.round += 1
                scores = list(ev["scores"])
                declared = accepted = others_declared = False
                oya, jun, calls = ev["oya"], 0, 0
                st.oya += oya == me
            elif ty == "dahai":
                jun += ev["actor"] == me
            elif ty in ("chi", "pon", "daiminkan"):
                calls += ev["actor"] == me
            elif ty == "reach":
                if ev["actor"] == me:
                    declared = True
                    st.riichi += 1
                    st.riichi_jun += jun
                    st.riichi_as_oya += oya == me
                    st.chasing_riichi += others_declared
                elif declared:
                    st.riichi_got_chased += 1
                else:
                    others_declared = True
            elif ty == "reach_accepted":
                scores[ev["actor"]] -= 1000
                accepted = accepted or ev["actor"] == me
            elif ty == "hora":
                deltas = ev["deltas"]
                scores = [a + b for a, b in zip(scores, deltas)]
                if ev["actor"] == me:
                    point = deltas[me] - 1000 * accepted  # the own stick comes back with the win and is not counted
                    st.agari += 1
                    st.agari_jun += jun
                    if oya == me:
                        st.agari_as_oya += 1
                        st.agari_point_oya += point
                    else:
                        st.agari_point_ko += point
                    if accepted:
                        st.riichi_agari += 1; st.riichi_agari_jun += jun; st.riichi_agari_point += point; st.riichi_point += point
                    elif calls > 0:
                        st.fuuro_agari += 1; st.fuuro_agari_jun += jun; st.fuuro_agari_point += point; st.fuuro_point += point
                    else:
                        st.dama_agari += 1; st.dama_agari_jun += jun; st.dama_agari_point += point
                    st.yakuman += point >= (48000 if oya == me else 32000)  # point.rs Point::yakuman(is_oya, 1).ron
                elif ev["target"] == me:
                    point = deltas[me]
                    st.houjuu += 1
                    st.houjuu_jun += jun
                    if oya == ev["actor"]:
                        st.houjuu_to_oya += 1
                        st.houjuu_point_to_oya += point
                    else:
                        st.houjuu_point_to_ko += point
                    if declared:
                        st.riichi_houjuu += 1; st.riichi_point += point
                    elif calls > 0:
                        st.fuuro_houjuu += 1; st.fuuro_point += point
            elif ty == "ryukyoku":
                deltas = ev["deltas"]
                scores = [a + b for a, b in zip(scores, deltas)]
                point = deltas[me]
                st.ryukyoku += 1
                st.ryukyoku_point += point
                if accepted:
                    st.riichi_ryukyoku += 1
                    st.riichi_point += point - 1000
                elif calls > 0:
                    st.fuuro_point += point
                st.nagashi_mangan += point >= 8000
            elif ty == "end_kyoku":
                if calls > 0:
                    st.fuuro += 1
                    st.fuuro_num += calls
        order = sorted(range(4), key=lambda i: -scores[i])  # rankings.rs:8-22, stable by seat
        total = sum(scores)
        if total < 100_000:  # sticks left on the table go to the top
            scores[order[0]] += 100_000 - total
        st.point = scores[me] - 25000
        st.tobi = int(scores[me] < 0)
        setattr(st, ("rank_1", "rank_2", "rank_3", "rank_4")[order.index(me)], 1)
        return st

    @staticmethod
    def from_log(log: str, player_id: int) -> "Stat":
        return Stat.from_game([json.loads(ln) for ln in log.splitlines() if ln.strip()], player_id)

    @staticmethod
    def from_dir(dir: str, player_name: str, disable_progress_bar: bool = False) -> "Stat":
        paths = _log_paths(dir)
        if _device_ready():
            return _device_from_dir(paths, player_name)
        total = Stat()
        for path in paths:
            total = total + _host_log_stat(path, player_name)
        return total

    def __repr__(self):
        return "Stat(" + ", ".join(f"{c}={getattr(self, c)}" for c in COUNTERS) + ")"

    def __str__(self):
        lines = [f"Games {self.game}", f"Rounds {self.round}", f"Rounds as dealer {self.oya}", ""]
        for k in (1, 2, 3, 4):
            lines.append(f"{k}{('st', 'nd', 'rd', 'th')[k - 1]} (rate) {getattr(self, f'rank_{k}')} ({getattr(self, f'rank_{k}_rate'):.6f})")
        lines += [f"Tobi(rate) {self.tobi} ({self.tobi_rate:.6f})", f"Avg rank {self.avg_rank:.6f}",
                  f"Total rank pt {self.total_pt([90, 45, 0, -135])}", f"Avg rank pt {self.avg_pt([90, 45, 0, -135]):.6f}",
                  f"Total score delta {self.point}", ""]
        lines += [f"{name} {getattr(self, name):.6f}" for name in RATES if not name.startswith("rank_") and name != "tobi_rate"]
        return "\n".join(lines)

    def reference_text(self) -> str:
        """the reference's report (the Display format of stat.rs:128-189): labels padded per block, Rust float formatting"""
        pt = [90, 45, 0, -135]
        blocks = [
            [("Games", self.game), ("Rounds", self.round), ("Rounds as dealer", self.oya)],
            [(f"{k}{('st', 'nd', 'rd', 'th')[k - 1]} (rate)", f"{getattr(self, f'rank_{k}')} ({_rs(getattr(self, f'rank_{k}_rate'))})")
             for k in (1, 2, 3, 4)]
            + [("Tobi(rate)", f"{self.tobi} ({_rs(self.tobi_rate)})"), ("Avg rank", _rs(self.avg_rank)),
               ("Total rank pt", self.total_pt(pt)), ("Avg rank pt", _rs(self.avg_pt(pt))), ("Total Δscore", self.point),
               ("Avg game Δscore", _rs(self.avg_point_per_game)), ("Avg round Δscore", _rs(self.avg_point_per_round))],
        ]
        blocks += [[(label, _rs(getattr(self, rate))) for label, rate in block] for block in _REFERENCE_RATES]
        blocks.append([("Yakuman (rate)", f"{self.yakuman} ({_rs(self.yakuman_rate, 9)})"),
                       ("Nagashi mangan (rate)", f"{self.nagashi_mangan} ({_rs(self.nagashi_mangan_rate, 9)})")])
        out = []
        for block in blocks:
            w = max(len(label) for label, _ in block)
            out.append("\n".join(f"{label.ljust(w)} {value}" for label, value in block))
        return "\n\n".join(out)


# the rate blocks of the reference's report (stat.rs:128-189), label -> derived quantity
_REFERENCE_RATES = (
    (("Win rate", "agari_rate"), ("Deal-in rate", "houjuu_rate"), ("Call rate", "fuuro_rate"), ("Riichi rate", "riichi_rate"),
     ("Ryukyoku rate", "ryukyoku_rate")),
    (("Avg winning Δscore", "avg_point_per_agari"), ("Avg winning Δscore as dealer", "avg_point_per_oya_agari"),
     ("Avg winning Δscore as non-dealer", "avg_point_per_ko_agari"),
     ("Avg riichi winning Δscore", "avg_point_per_riichi_agari"), ("Avg open winning Δscore", "avg_point_per_fuuro_agari"),
     ("Avg dama winning Δscore", "avg_point_per_dama_agari"), ("Avg ryukyoku Δscore", "avg_point_per_ryukyoku")),
    (("Avg winning turn", "avg_agari_jun"), ("Avg riichi winning turn", "avg_riichi_agari_jun"),
     ("Avg open winning turn", "avg_fuuro_agari_jun"), ("Avg dama winning turn", "avg_dama_agari_jun")),
    (("Avg deal-in turn", "avg_houjuu_jun"), ("Avg deal-in Δscore", "avg_point_per_houjuu"),
     ("Avg deal-in Δscore to dealer", "avg_point_per_houjuu_to_oya"),
     ("Avg deal-in Δscore to non-dealer", "avg_point_per_houjuu_to_ko")),
    (("Chasing riichi rate", "chasing_riichi_rate"), ("Riichi chased rate", "riichi_chased_rate"),
     ("Winning rate after riichi", "agari_rate_after_riichi"), ("Deal-in rate after riichi", "houjuu_rate_after_riichi"),
     ("Avg riichi turn", "avg_riichi_jun"), ("Avg riichi Δscore", "avg_riichi_point")),
    (("Avg number of calls", "avg_fuuro_num"), ("Winning rate after call", "agari_rate_after_fuuro"),
     ("Deal-in rate after call", "houjuu_rate_after_fuuro"), ("Avg call Δscore", "avg_fuuro_point")),
    (("Dealer wins/all dealer rounds", "agari_rate_as_oya"), ("Dealer wins/all wins", "agari_as_oya_rate"),
     ("Deal-in to dealer/all deal-ins", "houjuu_to_oya_rate")),
)


def _rs(x: float, prec: int = 6) -> str:
    """Rust's `{:.prec}` of an f64: Python's fixed-point digits, but `NaN`, `inf` and `-inf` for the non-finite values"""
    if math.isnan(x):
        return "NaN"
    if math.isinf(x):
        return "inf" if x > 0 else "-inf"
    return f"{x:.{prec}f}"


def _log_paths(dir: str):
    return glob.glob(os.path.join(dir, "**", "*.json"), recursive=True) + glob.glob(os.path.join(dir, "**", "*.json.gz"), recursive=True)


def _host_log_stat(path: str, player_name: str) -> Stat:
    """one log file on the host: json.loads of every line, then Stat.from_game for every seat named player_name"""
    opener = gzip.open if path.lower().endswith(".gz") else open
    with opener(path, "rt") as f:
        events = [json.loads(ln) for ln in f if ln.strip()]
    if not events or events[0].get("type") != "start_game":
        raise ValueError(f"first event is not start_game, got {events[0] if events else None!r}")
    total = Stat()
    for i, name in enumerate(events[0].get("names", [])):
        if name == player_name:
            total = total + Stat.from_game(events, i)
    return total


def _read_counters():
    """the counter names of include/mjx.h MJX_STAT_COUNTERS, in the order k_stat_logs writes them (the header is their single
    definition)"""
    from . import _cdecl

    return tuple(name for (name,) in _cdecl.xmacro(_cdecl.header(), "MJX_STAT_COUNTERS"))


def _seat_mask(blob: bytes, b: int, e: int, player_name: str):
    """the seats named player_name on a log's first event line (bytes [b, e)) as a bit mask, or None when the host must decide"""
    try:
        first = json.loads(blob[b:e].decode("utf-8"))
        if first.get("type") != "start_game":
            return None
        seats = [i for i, name in enumerate(first.get("names", [])) if name == player_name]
    except Exception:  # noqa: BLE001
        return None
    if any(i > 3 for i in seats):
        return None
    return sum(1 << i for i in seats)


def _chunks(paths, pool, step: int):
    """(paths, contents) of consecutive files in order, read + gunzipped on `pool` `step` at a time, cut at CHUNK_LOGS files or
    CHUNK_BYTES of text (a chunk always takes at least one file)"""
    return _logio.chunks(paths, pool, step, _read_bytes, CHUNK_LOGS, CHUNK_BYTES)


def _device_from_dir(paths, player_name: str, device: int | None = None) -> Stat:
    """from_dir on the device (default: _stat_device()): per chunk of files, read + gunzip on a thread pool, decode with the deltas
    output, k_stat_logs over the seats of every log, the counters summed on the device and copied back once; the rest of the
    chunk's files, in glob order, through _host_log_stat"""
    import numpy as np
    import torch

    from . import _lib
    from .validate_logs import decode_dev

    device = _stat_device() if device is None else device
    _lib.init(device)
    L = _lib.load()
    dev = torch.device("cuda", device)
    names = _read_counters()
    total = {c: 0 for c in COUNTERS}
    host_total = Stat()
    workers = min(32, os.cpu_count() or 1)
    # torch.cuda.device: the streams and allocations below belong to `device` whatever torch's current device is
    with torch.cuda.device(device), ThreadPoolExecutor(workers) as pool:  # zlib and file reads release the GIL
        for chunk, blobs in _chunks(paths, pool, 4 * workers):
            on_dev = [k for k, b in enumerate(blobs) if b is not None]
            host = [k for k, b in enumerate(blobs) if b is None]
            if on_dev:
                D = decode_dev([blobs[k] for k in on_dev], device, deltas=True)
                seats = np.zeros(len(on_dev), dtype=np.uint8)
                counted = []
                for j, k in enumerate(on_dev):
                    m = _seat_mask(blobs[k], int(D.counts[j, 4]), int(D.counts[j, 5]), player_name) if D.accept[j] else None
                    if m is None:
                        host.append(k)
                    else:
                        seats[j] = m; counted.append(j)
                n = len(on_dev)
                out = torch.empty((n, len(names)), dtype=torch.int64, device=dev)
                status = torch.empty(n, dtype=torch.int32, device=dev)
                d_seats = torch.from_numpy(seats).to(dev)
                ptr = lambda t: t.data_ptr() if t.numel() else None
                _lib.check(L.mjx_stat_logs_dev(n, ptr(D.hdr), D.offs[0].data_ptr(), D.offs[1].data_ptr(), D.hdr.numel(),
                                               ptr(D.kyoku), D.offs[2].data_ptr(), D.kyoku.numel(), ptr(D.deltas), ptr(D.has_deltas),
                                               d_seats.data_ptr(), out.data_ptr(), status.data_ptr(),
                                               torch.cuda.current_stream(dev).cuda_stream), "mjx_stat_logs_dev")
                # a log with a non-zero status has all-zero counters, so the sum counts exactly the logs with status 0
                res = torch.cat([out.sum(0), status.to(torch.int64)]).cpu().numpy()
                for name, v in zip(names, res[:len(names)]):
                    total[name] += int(v)
                st = res[len(names):]
                host += [on_dev[j] for j in counted if st[j] != 0]
            for k in sorted(host):
                host_total = host_total + _host_log_stat(chunk[k], player_name)
    return Stat(**total) + host_total


def main(argv=None) -> int:
    """bin/stat.rs: the report of Stat.from_dir(DIR, PLAYER_NAME) on stdout"""
    argv = sys.argv[1:] if argv is None else argv
    if len(argv) != 2:
        print("Usage: python -m mortal_b200.stat <DIR> <PLAYER_NAME>", file=sys.stderr)
        return 2
    try:
        st = Stat.from_dir(argv[0], argv[1], disable_progress_bar=True)
    except Exception as e:  # noqa: BLE001 — the reference's `Error: ...` exit
        print(f"Error: {type(e).__name__}: {e}", file=sys.stderr)
        return 1
    print(st.reference_text())
    return 0


if __name__ == "__main__":
    sys.exit(main())
