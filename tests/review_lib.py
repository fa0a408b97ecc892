"""Helpers of the review tests — TEST INFRASTRUCTURE: a deterministic stub engine and the per-line reference review (the Bot driven
as mortal.py's review mode drives it)."""
from __future__ import annotations

import re

import numpy as np

NONE_LINE = '{"type":"none","meta":{"mask_bits":0}}'
_EVAL = re.compile(r'"eval_time_ns":\d+')


def mask_eval(text: str) -> str:
    """the text with every meta.eval_time_ns set to 0 (the one field that is a measurement)"""
    return _EVAL.sub('"eval_time_ns":0', text)


def stub_q(obs: np.ndarray, masks: np.ndarray) -> np.ndarray:
    """Q-values of the stub, row by row: small integers from the observation's bits (its first 200 channels, none of them from the
    single-player block) and the mask, so ties are common; agari, kan and riichi are favoured, so the guard, kan_select and reach come up.
    Illegal actions get -inf. int64 arithmetic throughout: the same on the host and the device."""
    x = np.rint(obs[:, :200].reshape(len(obs), -1) * 8).astype(np.int64)
    w = np.arange(x.shape[1], dtype=np.int64) % 13 + 1
    s = (x * w).sum(1) + (masks.astype(np.int64) * (np.arange(46) + 1)).sum(1)
    a = np.arange(46, dtype=np.int64)
    q = ((s[:, None] * (a * 7 + 3) + a * 5) % 5).astype(np.float32) - 2
    q[:, 43] += 2
    q[:, 42] += 1
    q[:, 37] += 2
    return np.where(masks, q, -np.inf).astype(np.float32)


def first_argmax(q: np.ndarray) -> np.ndarray:
    return q.argmax(-1)


class StubEngine:
    """a host engine (react_batch only) computing stub_q"""
    engine_type = "mortal"
    is_oracle = False
    enable_quick_eval = False
    name = "stub"

    def __init__(self, guard: bool, version: int = 4):
        self.enable_rule_based_agari_guard = guard
        self.version = version

    def react_batch(self, obs, masks, invisible_obs):
        o = np.stack([np.asarray(x, dtype=np.float32) for x in obs])
        m = np.stack([np.asarray(x, dtype=bool) for x in masks])
        q = stub_q(o, m)
        return first_argmax(q).tolist(), q.tolist(), m.tolist(), [True] * len(q)


class DeviceStubEngine(StubEngine):
    """stub_q as torch int64 ops on the device (react_device), and the reference protocol over it"""

    def react_device(self, obs, masks, return_greedy=False):
        import torch

        x = torch.round(obs[:, :200].reshape(obs.shape[0], -1) * 8).to(torch.int64)
        w = torch.arange(x.shape[1], device=obs.device, dtype=torch.int64) % 13 + 1
        a = torch.arange(46, device=obs.device, dtype=torch.int64)
        s = (x * w).sum(1) + (masks.to(torch.int64) * (a + 1)).sum(1)
        q = ((s[:, None] * (a * 7 + 3) + a * 5) % 5).to(torch.float32) - 2
        q[:, 43] += 2
        q[:, 42] += 1
        q[:, 37] += 2
        q = q.masked_fill(~masks.bool(), -torch.inf)
        act = q.argmax(-1)
        if return_greedy:
            return act, q, torch.ones(q.shape[0], dtype=torch.bool, device=q.device)
        return act, q

    def react_batch(self, obs, masks, invisible_obs):
        import torch

        o = torch.as_tensor(np.stack(obs), device="cuda")
        m = torch.as_tensor(np.stack(masks), device="cuda")
        a, q, g = self.react_device(o, m, return_greedy=True)
        return a.tolist(), q.tolist(), m.tolist(), g.tolist()


def bot_review(engine, text: str, seat: int) -> str:
    """mortal.py review mode without the extra_data line: every non-empty stripped line to Bot.react, the reaction or the none line"""
    from mortal_b200.libriichi.mjai import Bot

    bot = Bot(engine, seat)
    out = []
    for ln in text.splitlines():
        ln = ln.strip()
        if ln:
            out.append((bot.react(ln) or NONE_LINE) + "\n")
    return "".join(out)


def emul_review(engine, event_logs, seats, version: int = 4):
    """The batched review on the host-emulated build (tests/host_emul/emul_review.cc), driven as mortal_b200.review drives the
    device: event_logs = lists of mjai events, seats = per log its seats -> list per job of (text or None, records dict, err, stopped
    event). The engine is a react_batch engine over host arrays (StubEngine)."""
    import emul_lib as E
    from mortal_b200 import dataset_codec as DC

    L = E.lib()
    assert L.emulr_init(E.DATA_DIR.encode()) == 0
    jobs = {k: np.ascontiguousarray(v) for k, v in DC.build_jobs(event_logs, seats).items()}
    n = len(jobs["players"])
    scan = np.zeros(n, dtype=np.int32)
    h = L.emulr_create(n, jobs["hdr"].ctypes.data, jobs["ev_off"].ctypes.data, jobs["ev_cnt"].ctypes.data, len(jobs["hdr"]),
                       jobs["kyoku"].ctypes.data, jobs["ky_off"].ctypes.data, len(jobs["kyoku"]), jobs["players"].ctypes.data,
                       scan.ctypes.data)
    rows = {1: 938, 2: 942, 3: 934, 4: 1012}[version]
    guard = int(bool(engine.enable_rule_based_agari_guard))
    cap = n * 3
    recs = []
    try:
        while True:
            live = L.emulr_step(h)
            rt = np.zeros(cap, np.int32); rs = np.zeros(cap, np.uint8); st = np.zeros(cap, np.uint32); m = np.zeros((cap, 46), np.uint8)
            nr = L.emulr_rows(h, rt.ctypes.data, rs.ctypes.data, st.ctypes.data, m.ctypes.data)
            if nr:
                obs = np.zeros((nr, rows, 34), dtype=np.float32)
                L.emulr_encode(h, obs.ctypes.data, version)
                actions, q, _, greedy = engine.react_batch(list(obs), list(m[:nr].astype(bool)), None)
                actions = np.ascontiguousarray(actions, dtype=np.int64)
                q = np.ascontiguousarray(q, dtype=np.float32)
                greedy = np.ascontiguousarray(greedy, dtype=np.uint8)
                info = np.zeros((nr, 4), np.int32); mask = np.zeros(nr, np.uint64); qo = np.zeros((nr, 46), np.float32)
                i64s = np.zeros((nr, 2), np.int64); word = np.zeros(nr, np.uint64)
                L.emulr_react(h, nr, actions.ctypes.data, q.ctypes.data, greedy.ctypes.data, guard, info.ctypes.data, mask.ctypes.data,
                              qo.ctypes.data, i64s.ctypes.data, word.ctypes.data)
                recs.append((rt[:nr].astype(np.int64), st[:nr].astype(np.int32), (rs[:nr] >> 2) & 1, info, mask, qo, i64s, word,
                             actions))
            if live == 0:
                break
        err = np.zeros(n, np.int32); stop = np.zeros(n, np.int32)
        L.emulr_results(h, err.ctypes.data, stop.ctypes.data)
    finally:
        L.emulr_destroy(h)
    cat = lambda k, shape, dt: np.concatenate([r[k] for r in recs]) if recs else np.zeros(shape, dt)
    job = cat(0, (0,), np.int64)
    order = np.argsort(job, kind="stable")
    job = job[order]
    event, kan, info, mask, qo, i64s, word, eng = (np.ascontiguousarray(cat(k, s, d)[order]) for k, s, d in
                                                   ((1, (0,), np.int32), (2, (0,), np.uint8), (3, (0, 4), np.int32),
                                                    (4, (0,), np.uint64), (5, (0, 46), np.float32), (6, (0, 2), np.int64),
                                                    (7, (0,), np.uint64), (8, (0,), np.int64)))
    rec_off = np.zeros(n + 1, np.int64)
    rec_off[1:] = np.cumsum(np.bincount(job, minlength=n))
    skip = (err != 0).astype(np.uint8)
    nbytes = np.zeros(n, np.int64)
    args = (n, jobs["ev_cnt"].ctypes.data, rec_off.ctypes.data, len(job), event.ctypes.data, kan.ctypes.data, word.ctypes.data,
            info.ctypes.data, mask.ctypes.data, qo.ctypes.data, i64s.ctypes.data, skip.ctypes.data)
    L.emulr_render(*args, nbytes.ctypes.data, None, None, 0)
    off = np.zeros(n + 1, np.int64)
    off[1:] = np.cumsum(nbytes)
    buf = np.zeros(max(int(off[-1]), 1), np.uint8)
    L.emulr_render(*args, None, off.ctypes.data, buf.ctypes.data, int(off[-1]))
    blob = buf.tobytes()
    out = []
    for j in range(n):
        sl = slice(int(rec_off[j]), int(rec_off[j + 1]))
        r = dict(event=event[sl], kan=kan[sl], info=info[sl], q=qo[sl], word=word[sl], engine_action=eng[sl])
        text = blob[int(off[j]):int(off[j + 1])].decode() if not err[j] else None
        out.append((text, r, int(err[j]), int(stop[j])))
    return out


def guard_logs(games):
    """(events, [seat]) variants of self-play games whose all-last kyoku (south 4) starts with `seat` far behind (1000 against
    33000 each), so that most agari of that seat would leave it fourth and the rule-based agari guard objects
    (agent_helper.rs:262-368). The scores are the only change; nothing downstream checks them against the deltas."""
    out = []
    for g in games:
        at = [i for i, e in enumerate(g) if e["type"] == "start_kyoku" and e["bakaze"] == "S" and e["kyoku"] == 4]
        if not at:
            continue
        i = at[-1]
        for p in range(4):
            if p == g[i]["oya"]:
                continue
            ev = [dict(e) for e in g]
            ev[i]["scores"] = [1000 if s == p else 33000 for s in range(4)]
            out.append((ev, [p]))
    return out


class IllegalStubEngine(StubEngine):
    """StubEngine that answers ryukyoku (44) where it is not legal on some rows (row-wise and deterministic): the reaction cannot
    be decoded there, so the Bot raises and the review fails that job at that event"""

    def react_batch(self, obs, masks, invisible_obs):
        actions, q, m, greedy = super().react_batch(obs, masks, invisible_obs)
        m_ = np.asarray(m, dtype=bool)
        qs = np.where(np.isfinite(q), np.asarray(q), 0).sum(1).astype(np.int64)
        bad = ~m_[:, 44] & (qs % 7 == 0)
        return [44 if b else a for a, b in zip(actions, bad)], q, m, greedy


class DeviceIllegalStubEngine(DeviceStubEngine):
    """IllegalStubEngine's rule as device ops"""

    def react_device(self, obs, masks, return_greedy=False):
        import torch

        act, q, g = super().react_device(obs, masks, return_greedy=True)
        qs = torch.where(torch.isfinite(q), q, torch.zeros_like(q)).sum(1).to(torch.int64)
        act = torch.where(~masks.bool()[:, 44] & (qs % 7 == 0), torch.full_like(act, 44), act)
        return (act, q, g) if return_greedy else (act, q)


def bot_fail_index(engine, text: str, seat: int):
    """the index of the line the Bot raises on (mortal.py would stop there), or None"""
    from mortal_b200.libriichi.mjai import Bot

    bot = Bot(engine, seat)
    lines = [ln.strip() for ln in text.splitlines() if ln.strip()]
    for i, ln in enumerate(lines):
        try:
            bot.react(ln)
        except Exception:  # noqa: BLE001 — the Bot's failure is the point
            return i
    return None
