"""Review mjai logs with a Mortal engine: what `MORTAL_REVIEW_MODE=1 python mortal.py <seat>` prints for a log, for a whole batch of
logs and seats in one device pass (csrc/mjx_review.cuh, include/mjx_review.h).

    reviews = review_logs(engine, logs, player_ids, grp=None, model_tag=None)
    reviews[i][k].player_id, .text, .error, and per decision .event_index, .action, .label, .q_values, .masks, .is_greedy

The spec is libriichi.mjai.Bot fed every non-empty stripped line of the log, printing its reaction or the `none` line, then the
extra_data line (with `grp`). The batched path: the texts staged and gunzipped on the device (_logio.stage), decoded
(decode_dev_text), replayed in review mode (every event applied, a stop at every event where the seat can act), encoded, the engine
called on all decisions of a step at once, the reaction kernel (agari guard + decode), and the text rendered on the device. Logs the
decoder declines, logs that are not UTF-8 and logs whose lines carry `can_act` go through the Bot itself, with the same result.

    python -m mortal_b200.review DIR PLAYER_NAME OUT_DIR   reviews every .json / .json.gz log in DIR where PLAYER_NAME sits
"""
from __future__ import annotations

import gzip
import inspect
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import _cdecl, _lib, _logio

HEADER = os.path.join(os.path.dirname(_cdecl.HEADER), "mjx_review.h")
with open(HEADER) as _f:
    SYMBOLS = _cdecl.functions(_f.read(), "mjx_")  # the entries of include/mjx_review.h, exported by libmjx.so
_FLAGS = _cdecl.enum(_cdecl.header(), "mjx_mw_rec_flag")
_GREEDY = _FLAGS["MJX_MW_REC_GREEDY"]
NONE_LINE = '{"type":"none","meta":{"mask_bits":0}}'
_BOUND = None


def _load():
    global _BOUND
    if _BOUND is None:
        _BOUND = _cdecl.bind(_lib.load(), SYMBOLS)
    return _BOUND


class Review:
    """The review of one (log, seat). text: the review's lines, each ending in "\\n" (None when the log failed, error then says
    where). The per-decision fields are device tensors, one entry per event where the seat could act, in event order; q_values
    and masks are those of the decision row (a kan-select row's are in the text's meta only)."""

    def __init__(self, player_id, text=None, error=None, event_index=None, action=None, label=None, q_values=None, masks=None,
                 is_greedy=None):
        self.player_id, self.text, self.error = player_id, text, error
        self.event_index, self.action, self.label = event_index, action, label
        self.q_values, self.masks, self.is_greedy = q_values, masks, is_greedy


def check_engine(engine) -> None:
    """the engines a review takes: a Bot's (engine_type 'mortal', not an oracle) that evaluates every decision"""
    if getattr(engine, "engine_type", None) != "mortal":
        raise ValueError(f"unknown engine type {getattr(engine, 'engine_type', None)!r}")
    if getattr(engine, "is_oracle", False):
        raise ValueError("an oracle engine needs the invisible state, which a reviewer never has (mortal.rs:253-255)")
    if getattr(engine, "enable_quick_eval", True):
        raise ValueError("review needs enable_quick_eval=False: every decision is evaluated and reported")


def _is_path(x) -> bool:
    if isinstance(x, os.PathLike):
        return True
    return isinstance(x, str) and "\n" not in x and x.lower().endswith((".json", ".json.gz"))


def _bot_review(engine, text: str, seat: int):
    """the Bot fed line by line as mortal.py review mode feeds it -> (text, error)"""
    from .libriichi.mjai import Bot

    bot = Bot(engine, seat)
    out = []
    lines = [ln.strip() for ln in text.splitlines()]
    lines = [ln for ln in lines if ln]
    for e, ln in enumerate(lines):
        try:
            r = bot.react(ln)
        except Exception as exc:  # noqa: BLE001 — the review of this log fails; the others go on
            return None, f"seat {seat}: event {e}: {exc}"
        out.append((r or NONE_LINE) + "\n")
    return "".join(out), None


def _react_fn(engine):
    """engine rows -> (actions int64, q float32 [n, 46], is_greedy bool) on the device"""
    import torch

    rd = getattr(engine, "react_device", None)
    if rd is not None and "return_greedy" in inspect.signature(rd).parameters:
        def react(obs, masks):
            a, q, g = rd(obs, masks, return_greedy=True)
            return a.long(), q.float(), g.bool()
        return react

    def react(obs, masks):  # the reference protocol: lists of per-row arrays in, lists out
        dev = obs.device
        actions, q, _, greedy = engine.react_batch(list(obs.cpu().numpy()), list(masks.cpu().numpy()), None)
        return (torch.as_tensor(np.asarray(actions, dtype=np.int64), device=dev),
                torch.as_tensor(np.asarray(q, dtype=np.float32), device=dev),
                torch.as_tensor(np.asarray(greedy, dtype=bool), device=dev))
    return react


def _review_device(engine, D, slots, seats, device):
    """the review of log slot slots[i] of D for seats seats[i] -> list (per job) of (Review, failed event or None, error code)"""
    import torch

    from .env import ReplayEnv

    dev = torch.device("cuda", device)
    ev_off, ev_cnt, ky_off, pids = [], [], [], []
    for s, ps in zip(slots, seats):
        for p in ps:
            ev_off.append(int(D.ev_off[s])); ev_cnt.append(int(D.ev_cnt[s])); ky_off.append(int(D.ky_off[s])); pids.append(p)
    n_jobs = len(pids)
    jobs = dict(hdr=D.hdr, kyoku=D.kyoku, ev_off=np.array(ev_off, dtype=np.int32), ev_cnt=np.array(ev_cnt, dtype=np.int32),
                ky_off=np.array(ky_off, dtype=np.int32), players=np.array(pids, dtype=np.uint8))
    version = int(getattr(engine, "version", 4))
    guard = int(bool(getattr(engine, "enable_rule_based_agari_guard", False)))
    react = _react_fn(engine)
    R = _load()
    env = ReplayEnv(jobs, obs_version=version, device=device)
    steps = []
    try:
        st = lambda: torch.cuda.current_stream(dev).cuda_stream
        _lib.check(R.mjx_env_replay_review(env._h, st()), "mjx_env_replay_review")
        while True:
            env.replay_step()
            nr = env.num_rows()
            if nr:
                obs = env.encode_obs()[:nr]
                masks = env.masks[:nr]
                t0 = time.perf_counter_ns()
                actions, q, greedy = react(obs, masks)
                torch.cuda.synchronize(dev)
                eval_ns = time.perf_counter_ns() - t0
                actions, q, greedy = actions.contiguous(), q.contiguous(), greedy.to(torch.uint8).contiguous()
                kan = (env.row_seat[:nr] >> 2) & 1
                info = torch.empty((nr, 4), dtype=torch.int32, device=dev)
                mask = torch.empty(nr, dtype=torch.int64, device=dev)
                qo = torch.empty((nr, 46), dtype=torch.float32, device=dev)
                i64s = torch.empty((nr, 2), dtype=torch.int64, device=dev)
                word = torch.empty(nr, dtype=torch.int64, device=dev)
                _lib.check(R.mjx_review_react_dev(env._h, nr, actions.data_ptr(), q.data_ptr(), greedy.data_ptr(), guard,
                                                  info.data_ptr(), mask.data_ptr(), qo.data_ptr(), i64s.data_ptr(), word.data_ptr(),
                                                  st()), "mjx_review_react_dev")
                n_dec = nr - int(kan.sum())  # mortal.py's eval_time_ns: the engine call's time over its decisions
                i64s[:, 1] = eval_ns // max(n_dec, 1)
                steps.append((env.row_table[:nr].long(), env.row_step[:nr].to(torch.int32), kan.to(torch.uint8), info, mask, qo,
                              i64s, word))
            if env.num_live() == 0:
                break
        res = env.results()
        sp_overflows = env.sp_overflows() if version == 4 else 0
    finally:
        env.close()
    if sp_overflows:
        raise RuntimeError(f"single-player state arena overflowed in {sp_overflows} replay step(s): observation rows 889-1011 "
                           "would be zero; review fewer logs per call")
    cat = lambda k, dt: torch.cat([s[k] for s in steps]) if steps else torch.zeros(0, dtype=dt, device=dev)
    job = cat(0, torch.int64)
    order = torch.sort(job, stable=True).indices  # a job's records stay in event order, a kan-select row after its decision row
    job = job[order]
    event, kan, info, mask, qo, i64s, word = (cat(k, dt)[order].contiguous() for k, dt in
                                              ((1, torch.int32), (2, torch.uint8), (3, torch.int32), (4, torch.int64),
                                               (5, torch.float32), (6, torch.int64), (7, torch.int64)))
    counts = torch.bincount(job, minlength=n_jobs)
    rec_off = torch.zeros(n_jobs + 1, dtype=torch.int64, device=dev)
    rec_off[1:] = torch.cumsum(counts, 0)
    err = res["err"]
    skip = torch.from_numpy((err != 0).astype(np.uint8)).to(dev)
    d_cnt = torch.from_numpy(jobs["ev_cnt"]).to(dev)
    ptr = lambda t: t.data_ptr() if t.numel() else None
    recs = (int(job.numel()), ptr(event), ptr(kan), ptr(word), ptr(info), ptr(mask), ptr(qo), ptr(i64s), skip.data_ptr())
    nbytes = torch.empty(n_jobs, dtype=torch.int64, device=dev)
    _lib.check(R.mjx_review_render_count_dev(n_jobs, d_cnt.data_ptr(), rec_off.data_ptr(), *recs, nbytes.data_ptr(),
                                             torch.cuda.current_stream(dev).cuda_stream), "mjx_review_render_count_dev")
    off = torch.zeros(n_jobs + 1, dtype=torch.int64, device=dev)
    off[1:] = torch.cumsum(nbytes, 0)
    off_h = off.cpu().numpy()
    total = int(off_h[-1])
    out = torch.empty(max(total, 1), dtype=torch.uint8, device=dev)
    _lib.check(R.mjx_review_render_fill_dev(n_jobs, d_cnt.data_ptr(), rec_off.data_ptr(), *recs, off.data_ptr(), out.data_ptr(), total,
                                            torch.cuda.current_stream(dev).cuda_stream), "mjx_review_render_fill_dev")
    blob = out[:total].cpu().numpy().tobytes()
    main = kan == 0
    m_job = job[main]
    m_off = [0] + torch.cumsum(torch.bincount(m_job, minlength=n_jobs), 0).tolist()
    m_event, m_info, m_q = event[main], info[main], qo[main]
    m_masks = ((mask[main].unsqueeze(1) >> torch.arange(46, device=dev)) & 1).bool()
    last_event = {}
    if (err != 0).any():  # the event a failed job stopped at: the replay's (mjx_env_results steps in review mode)
        last_event = {j: int(res["steps"][j]) for j in np.nonzero(err)[0]}
    out_jobs = []
    for j in range(n_jobs):
        sl = slice(m_off[j], m_off[j + 1])
        rv = Review(pids[j], event_index=m_event[sl], action=m_info[sl, 0], label=m_info[sl, 3], q_values=m_q[sl],
                    masks=m_masks[sl], is_greedy=(m_info[sl, 1] & _GREEDY) != 0)
        if err[j] == 0:
            rv.text = blob[int(off_h[j]):int(off_h[j + 1])].decode("utf-8")
        out_jobs.append((rv, last_event.get(j), int(err[j])))
    return out_jobs


def review_logs(engine, logs, player_ids, grp=None, model_tag=None, *, device=None):
    """logs: texts, or paths of .json / .json.gz files; player_ids: per log a seat or a list of seats -> list (per log) of list (per
    seat) of Review. With `grp` (a GRP module or its state dict) every text ends with mortal.py's extra_data line: model_tag and the
    rank-probability matrix after every kyoku."""
    import torch

    check_engine(engine)
    if device is None:
        device = _logio.log_device()
    logs = list(logs)
    seats = [[int(p)] if isinstance(p, (int, np.integer)) else [int(x) for x in p] for p in player_ids]
    if len(seats) != len(logs):
        raise ValueError(f"{len(logs)} logs but {len(seats)} player_ids entries")
    for ps in seats:
        if any(not 0 <= p <= 3 for p in ps):
            raise ValueError("player_id must be within 0..3")
    names = [os.fspath(lg) if _is_path(lg) else f"log {i}" for i, lg in enumerate(logs)]
    results = [[None] * len(ps) for ps in seats]
    features = [None] * len(logs)
    texts = {}  # host texts of the logs the Bot reviews

    def host_text(i):
        if i not in texts:
            lg = logs[i]
            if _is_path(lg):
                p = os.fspath(lg)
                texts[i] = _logio.host_text(_logio.read_gz(p) if p.lower().endswith(".gz") else open(p, "rb").read())
            else:
                texts[i] = lg
        return texts[i]

    def read(i):  # the chunk reader: a file's raw bytes, or a text's UTF-8 bytes (None: not UTF-8, the Bot decides)
        lg = logs[i]
        if _is_path(lg):
            return _logio.read_file(os.fspath(lg))
        try:
            return lg.encode("utf-8"), False
        except UnicodeEncodeError:
            return None, False

    with torch.cuda.device(device), ThreadPoolExecutor(max(1, min(32, os.cpu_count() or 1))) as pool:
        _lib.init(device)
        from .dataset import _grp_run
        from .validate_logs import decode_dev_text

        for idx, items in _logio.chunks(list(range(len(logs))), pool, 256, read, _logio.CHUNK_LOGS, _logio.CHUNK_BYTES,
                                        _logio.text_size):
            T = _logio.stage(items, device, pool)
            slot = {idx[k]: j for j, k in enumerate(T.files)}
            D = decode_dev_text(T.text, T.log_off, device, deltas=grp is not None, status=T.status)
            can_act = _logio.count_keys(T.text, T.log_off, [b'"can_act"'], device)[:, 0] if T.files else np.zeros(0, np.int64)
            on_dev = [i for i in idx if i in slot and D.accept[slot[i]] and can_act[slot[i]] == 0]
            if on_dev:
                for i, (rv, ev, code) in zip([i for i in on_dev for _ in seats[i]],
                                             _review_device(engine, D, [slot[i] for i in on_dev], [seats[i] for i in on_dev], device)):
                    k = sum(1 for r in results[i] if r is not None)
                    if code:
                        rv.error = f"{names[i]}: seat {rv.player_id}: replay failed at event {ev} with mjx error code {code}"
                    results[i][k] = rv
                if grp is not None:
                    G = _grp_run(D, device)
                    for i in on_dev:
                        g = G.grp(D, slot[i])
                        features[i] = g.take_feature() if g is not None else None
            dev_set = set(on_dev)
            for i in idx:
                if i in dev_set:
                    continue
                for k, p in enumerate(seats[i]):
                    try:
                        text, error = _bot_review(engine, host_text(i), p)
                    except Exception as exc:  # noqa: BLE001 — an unreadable log fails its review only
                        text, error = None, f"seat {p}: {exc}"
                    results[i][k] = Review(p, text=text, error=None if error is None else f"{names[i]}: {error}")
        if grp is not None:
            from .dataset import Grp
            from .reward import RewardCalculator

            todo = []
            for i in range(len(logs)):
                if all(r.text is None for r in results[i]):
                    continue
                try:
                    if features[i] is None:  # GRP features the device declined, or a log the Bot reviewed
                        features[i] = Grp.load_log(host_text(i)).take_feature()
                    if len(features[i]) == 0:
                        raise ValueError("the log has no kyoku")
                    todo.append(i)
                except Exception as exc:  # noqa: BLE001 — no rank-probability matrix: this log's review fails, the others go on
                    for r in results[i]:
                        if r.text is not None:
                            r.text, r.error = None, f"{names[i]}: seat {r.player_id}: GRP features: {exc}"
            if todo:
                rc = RewardCalculator(grp, device=device)
                matrix = rc._launch([np.asarray(features[i], dtype=np.float64) for i in todo])[0].cpu().numpy()  # one launch
                at = 0
                for i in todo:
                    m = matrix[at:at + len(features[i])]
                    at += len(features[i])
                    extra = json.dumps({"model_tag": model_tag, "phi_matrix": m.tolist()}) + "\n"
                    for r in results[i]:
                        if r.text is not None:
                            r.text += extra
    return results


def main(argv=None) -> int:
    argv = sys.argv[1:] if argv is None else argv
    if len(argv) != 3:
        print("Usage: python -m mortal_b200.review <DIR> <PLAYER_NAME> <OUT_DIR>", file=sys.stderr)
        return 1
    src, name, out_dir = argv
    from .mortal import load_review_engine

    engine, grp, tag = load_review_engine()
    files = sorted(f for f in os.listdir(src) if f.lower().endswith((".json", ".json.gz")))
    paths, seats, unreadable = [], [], 0
    for f in files:
        p = os.path.join(src, f)
        try:  # the names are on the first line: only that much is read here
            with (gzip.open(p, "rb") if f.lower().endswith(".gz") else open(p, "rb")) as fh:
                first = json.loads(fh.readline().decode("utf-8"))
            ps = [s for s, nm in enumerate(first.get("names", [])) if nm == name]
        except Exception as exc:  # noqa: BLE001 — an unreadable file is reported and skipped
            print(f"{p}: {exc}", file=sys.stderr)
            unreadable += 1
            continue
        if ps:
            paths.append(p); seats.append(ps)
    reviews = review_logs(engine, paths, seats, grp=grp, model_tag=tag)
    os.makedirs(out_dir, exist_ok=True)
    n_dec = n_lab = n_match = failed = 0
    for p, rs in zip(paths, reviews):
        stem = os.path.basename(p)
        stem = stem[:-len(".json.gz")] if stem.lower().endswith(".json.gz") else stem[:-len(".json")]
        bad = False
        for r in rs:
            if r.error is not None:
                print(r.error, file=sys.stderr)
                bad = True
                continue
            with open(os.path.join(out_dir, f"{stem}.{r.player_id}.jsonl"), "w") as f:
                f.write(r.text)
            if r.action is not None:
                n_dec += int(r.action.numel())
                lab = r.label >= 0
                n_lab += int(lab.sum())
                n_match += int(((r.action == r.label) & lab).sum())
        failed += bad
    print(json.dumps({"logs": len(paths), "decisions": n_dec, "labelled": n_lab, "matching": n_match,
                      "failed": failed + unreadable}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
