"""Arena mjai logs rendered on the device (csrc/mjx_mjai_write.cuh): the environment's event words, its per-step log lengths and the
per-decision meta records become the log text in one count and one fill pass per chunk, then gzip files written on a thread pool.

The output is byte for byte what mortal_b200.mjai_log.write_logs writes (decode_events + attach_meta + dump_json_log): the start_game
and end_game lines are rendered here with the host writer's json.dumps, everything between them on the device. A game the host writer
would raise on gets a non-zero status, and the caller hands the whole part to the host writer, which raises the same exception.
"""
from __future__ import annotations

import ctypes as C
import gzip
import os

import numpy as np

from . import _lib, mjai_log

CHUNK_BYTES = 256 << 20  # text rendered and copied back per fill pass (consecutive games; a longer game goes alone)


def recorder_records(rec):
    """The meta records of a libriichi.arena._MetaRecorder as arrays, built from exactly what its finish() reads — without the
    per-row dicts. Returns (bounds int32 [n_steps, n_games], recs dict) or raises the recorder's error as finish() does."""
    if rec.error is not None:
        raise rec.error
    bounds = np.array(rec.bounds, dtype=np.int32).reshape(len(rec.bounds), rec.n)
    cols = {k: [] for k in ("table", "cycle", "seat", "kan", "action", "mask", "q", "i64", "flags", "shanten", "row")}
    row_base = 0
    weights = np.left_shift(np.uint64(1), np.arange(46, dtype=np.uint64))
    for cycle, tbl, rs, act, masks, sh, fu in rec.rows:
        nr = len(tbl)
        q_rows = np.zeros((nr, 46), dtype=np.float32)
        batch, ns = np.zeros(nr, dtype=np.int64), np.zeros(nr, dtype=np.int64)
        greedy = np.ones(nr, dtype=bool)
        for idx, q, eval_ns, g in rec.q.get(cycle, []):
            q_rows[idx] = q
            batch[idx] = len(idx)
            ns[idx] = eval_ns
            if g is not None:
                greedy[idx] = g
        rs = np.asarray(rs).astype(np.int64)
        flags = greedy.astype(np.int32)
        if sh is not None:
            flags |= 2
        if fu is not None:
            flags |= 4 | (np.asarray(fu, dtype=bool).astype(np.int32) << 3)
        cols["table"].append(np.asarray(tbl, dtype=np.int64))
        cols["cycle"].append(np.full(nr, cycle, dtype=np.int64))
        cols["seat"].append(rs & 3)
        cols["kan"].append((rs >> 2) & 1)
        cols["action"].append(np.asarray(act, dtype=np.int64))
        cols["mask"].append((np.asarray(masks, dtype=bool).astype(np.uint64) * weights).sum(1, dtype=np.uint64))
        cols["q"].append(q_rows)
        cols["i64"].append(np.stack([batch, ns], axis=1))
        cols["flags"].append(flags)
        cols["shanten"].append(np.zeros(nr, dtype=np.int64) if sh is None else np.asarray(sh, dtype=np.int64))
        cols["row"].append(np.arange(row_base, row_base + nr, dtype=np.int64))
        row_base += nr
    if not row_base:
        return bounds, None
    c = {k: np.concatenate(v) for k, v in cols.items()}
    return bounds, c


class DeviceMetaRecorder:
    """_MetaRecorder's records kept on the device: per environment step a device copy of log_len, per agent call one
    mjx_meta_record_dev launch appending a record per decision row (k_meta_record). Nothing is copied to the host and nothing
    synchronises while the games run; the (batch_size, eval_time_ns) of every call are host values uploaded once at the end.
    Capacity grows between launches (the row count of a call is known on the host); a launch never writes past it.
    A record is 221 bytes: table 4, cycle 4, seat 1, action/flags/shanten/row 16, mask 8, Q-values 184, call 4."""

    def __init__(self, n_games: int, version: int, env):
        import torch

        self.torch, self.n, self.version, self.env = torch, n_games, version, env
        self.dev = env.device
        self.error = None  # as in _MetaRecorder: the metadata is optional, a failure never takes the game loop down
        self.n_steps, self.count, self.calls, self.max_cycle = 0, 0, [], -1
        self.bounds = torch.zeros((64, n_games), dtype=torch.int32, device=self.dev)
        self._alloc(max(4 * env.row_cap, 1 << 14))

    def _alloc(self, cap):
        t, dev = self.torch, self.dev
        new = dict(table=t.empty(cap, dtype=t.int32, device=dev), cycle=t.empty(cap, dtype=t.int32, device=dev),
                   seat=t.empty(cap, dtype=t.uint8, device=dev), info=t.empty((cap, 4), dtype=t.int32, device=dev),
                   mask=t.empty(cap, dtype=t.int64, device=dev), q=t.empty((cap, 46), dtype=t.float32, device=dev),
                   call=t.empty(cap, dtype=t.int32, device=dev))
        if self.count:
            for k, v in new.items():
                v[:self.count].copy_(self.rec[k][:self.count])
        self.rec, self.cap = new, cap

    def _guard(fn):
        def wrapped(self, *a, **k):
            if self.error is not None:
                return None
            try:
                return fn(self, *a, **k)
            except Exception as exc:
                self.error = exc
                return None
        return wrapped

    @_guard
    def add_bounds(self, log_len_dev):
        if self.n_steps == self.bounds.shape[0]:
            self.bounds = self.torch.cat([self.bounds, self.torch.zeros_like(self.bounds)])
        self.bounds[self.n_steps].copy_(log_len_dev)
        self.n_steps += 1

    def new_call(self, n_rows, eval_ns):
        self.calls.append((int(n_rows), int(eval_ns)))
        return len(self.calls) - 1

    @_guard
    def record(self, cycle, n, q, actions, *, idx=None, greedy=None, call_ids=None, call=0, obs=None):
        """k_meta_record over the n rows of an agent call: q [n, 46] device, actions int64 [row_cap] device (the decisions taken),
        idx int64 [n] device (None: rows 0..n-1), greedy bool [n] device or None, call_ids int32 [n] device or None (every row:
        `call`), obs the v4 observation buffer [row_cap, rows, 34] or None"""
        import ctypes as C

        t, env = self.torch, self.env
        if n == 0:
            return
        if self.count + n > self.cap:
            self._alloc(max(2 * self.cap, self.count + n))
        q = q.float().contiguous()
        ptr = lambda x: None if x is None else C.c_void_p(x.data_ptr())
        g = None if greedy is None else greedy.to(t.uint8).contiguous()
        idx = None if idx is None else idx.to(t.int64).contiguous()
        use_obs = obs if self.version == 4 else None
        R = self.rec
        _lib.check(_lib.load().mjx_meta_record_dev(
            n, ptr(idx), ptr(q), ptr(g), ptr(call_ids), int(call), int(cycle), ptr(env.row_table), ptr(env.row_seat),
            ptr(actions), ptr(env.masks), ptr(use_obs), 0 if use_obs is None else int(use_obs.shape[1]), env.row_cap,
            ptr(R["table"]), ptr(R["cycle"]), ptr(R["seat"]), ptr(R["info"]), ptr(R["mask"]), ptr(R["q"]), ptr(R["call"]),
            self.count, self.cap, C.c_void_p(t.cuda.current_stream(self.dev).cuda_stream)), "mjx_meta_record_dev")
        self.count += n
        self.max_cycle = max(self.max_cycle, int(cycle))

    def device_args(self):
        """the renderer's arguments as device tensors, sorted on the device (raises the recording error, as finish() does)"""
        t = self.torch
        if self.error is not None:
            raise self.error
        n = self.count
        if not n or not self.n_steps:
            return None
        R = {k: v[:n] for k, v in self.rec.items()}
        key_steps = max(self.n_steps, self.max_cycle + 1)
        seat = R["seat"].long()
        key = ((R["table"].long() * key_steps + R["cycle"].long()) * 4 + (seat & 3)) * 2 + ((seat >> 2) & 1)
        order = t.argsort(key, stable=True)  # equal keys keep their order: the renderer takes the last one
        calls = t.tensor(self.calls, dtype=t.int64).reshape(-1, 2).to(self.dev, non_blocking=True)
        call = R["call"][order].long()
        i64 = t.where((call >= 0).unsqueeze(1), calls[call.clamp(min=0)], t.zeros((), dtype=t.int64, device=self.dev))
        return dict(bounds=self.bounds[:self.n_steps].contiguous(), n_steps=self.n_steps, key_steps=key_steps, key=key[order].contiguous(),
                    info=R["info"][order].contiguous(), mask=R["mask"][order].contiguous(), q=R["q"][order].contiguous(),
                    i64=i64.contiguous(), n_rec=n)

    def finish(self):
        """(bounds, decisions) as _MetaRecorder.finish returns them, from a host copy of the records (the host writer's input
        when a part falls back to it)"""
        from .mjai_log import make_meta

        if self.error is not None:
            raise self.error
        bounds = self.bounds[:self.n_steps].cpu().numpy()
        decisions = [dict() for _ in range(self.n)]
        n = self.count
        if not n:
            return bounds, decisions
        R = {k: v[:n].cpu().numpy() for k, v in self.rec.items()}
        order = np.lexsort((R["info"][:, 3], R["cycle"], R["table"]))  # per (table, cycle) in row order, as add_rows saw them
        pos = {}
        for i in order:
            pos[(int(R["table"][i]), int(R["cycle"][i]), int(R["seat"][i]) & 3, bool(R["seat"][i] & 4))] = i
        weights = 1 << np.arange(46, dtype=np.int64)

        def meta(i, m, kan_select=None):
            b, ns = self.calls[R["call"][m]] if R["call"][m] >= 0 else (0, 0)
            fl = int(R["info"][m, 1])
            legal = (int(R["mask"][i]) & weights) != 0
            return make_meta(int(R["info"][i, 0]), legal, R["q"][i], is_greedy=bool(R["info"][i, 1] & 1), batch_size=b, eval_time_ns=ns,
                             shanten=int(R["info"][m, 2]) if fl & 2 else None, at_furiten=bool(fl & 8) if fl & 4 else None,
                             kan_select=kan_select)
        for (tb, cy, seat, kan), i in pos.items():
            if kan or tb < 0:
                continue
            kan_meta = None
            kr = pos.get((tb, cy, seat, True))
            if kr is not None and int(R["info"][i, 0]) == 42:
                km = meta(kr, i)
                kan_meta = {k: v for k, v in km.items() if not k.startswith("_") and v is not None}
            decisions[tb].setdefault(cy, {})[seat] = meta(i, i, kan_meta)
        return bounds, decisions


def render_args(bounds, recs):
    """The record arrays of mjx_mjai_render_*_dev (host numpy, sorted by key) from recorder_records' output."""
    if bounds is None or recs is None or not len(recs["table"]) or not len(bounds):
        return dict(bounds=None, n_steps=0, key_steps=1, key=None, info=None, mask=None, q=None, i64=None, n_rec=0)
    n_steps = int(bounds.shape[0])
    key_steps = max(n_steps, int(recs["cycle"].max()) + 1)
    key = ((recs["table"] * key_steps + recs["cycle"]) * 4 + recs["seat"]) * 2 + recs["kan"]
    order = np.argsort(key, kind="stable")  # equal keys keep their row order: the renderer takes the last, as finish()'s dict does
    info = np.stack([recs["action"], recs["flags"], recs["shanten"], recs["row"]], axis=1).astype(np.int32)
    return dict(bounds=np.ascontiguousarray(bounds, dtype=np.int32), n_steps=n_steps, key_steps=key_steps,
                key=np.ascontiguousarray(key[order], dtype=np.int64), info=np.ascontiguousarray(info[order]),
                mask=np.ascontiguousarray(recs["mask"][order], dtype=np.uint64),
                q=np.ascontiguousarray(recs["q"][order], dtype=np.float32),
                i64=np.ascontiguousarray(recs["i64"][order], dtype=np.int64), n_rec=int(len(order)))


def _heads(names_per_game, seeds):
    """the start_game and end_game lines of every game, as mjai_log.dump_json_log renders them"""
    out = []
    for names, seed in zip(names_per_game, seeds):
        text = mjai_log.dump_json_log([], names, seed)
        k = text.index("\n") + 1  # json.dumps escapes line breaks: the first "\n" ends the start_game line
        out.append((text[:k].encode("utf-8"), text[k:].encode("utf-8")))
    return out


def _write_gz(path, head, body, tail):
    with gzip.open(path, "wb", compresslevel=9) as f:
        f.write(head + bytes(body) + tail)


def write_logs_device(log_dir, env, seeds, names_per_game, split_names, pool, bounds=None, recs=None, timing=None, dev_args=None):
    """mjai_log.write_logs over a CUDA BatchEnv's device log; returns the paths, or None when a game's words are something the host
    writer raises on (the caller then runs the host writer, which raises). `timing` (a dict) receives the stage times in seconds."""
    import time

    import torch

    n, cap = env.n_tables, env._log_cap
    dev = env.device
    stream = torch.cuda.current_stream(dev)
    sp = C.c_void_p(stream.cuda_stream)
    L = _lib.load()
    lens_h = env.log_len.cpu().numpy()
    if (lens_h > cap).any():  # BatchEnv.read_log's check and message
        raise RuntimeError(f"event log overflow: {int(lens_h.max())} words > capacity {cap}")
    try:
        heads = _heads(names_per_game, seeds)
    except Exception:  # noqa: BLE001 — e.g. a name that cannot be encoded: the host writer raises it at that game
        return None
    t0 = time.perf_counter()
    if dev_args is not None:  # records kept on the device (DeviceMetaRecorder)
        a = dv = dev_args
    else:
        a = render_args(bounds, recs)
        dv = {k: (torch.from_numpy(v.view(np.int64) if v.dtype == np.uint64 else v).to(dev, non_blocking=False)
                  if isinstance(v, np.ndarray) else None) for k, v in a.items()}
    ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    common = (n, C.c_void_p(env.log_words.data_ptr()), C.c_void_p(env.log_len.data_ptr()), cap, ptr(dv["bounds"]), a["n_steps"],
              a["key_steps"], ptr(dv["key"]), ptr(dv["info"]), ptr(dv["mask"]), ptr(dv["q"]), ptr(dv["i64"]), a["n_rec"])
    nbytes = torch.empty(n, dtype=torch.int32, device=dev)
    status = torch.empty(n, dtype=torch.int32, device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)] if timing is not None else None
    if ev:
        ev[0].record(stream)
    _lib.check(L.mjx_mjai_render_count_dev(*common, C.c_void_p(nbytes.data_ptr()), C.c_void_p(status.data_ptr()), sp),
               "mjx_mjai_render_count_dev")
    if ev:
        ev[1].record(stream)
    nb_h, st_h = nbytes.cpu().numpy(), status.cpu().numpy()
    if (st_h != 0).any():
        return None
    off_h = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(nb_h, out=off_h[1:])
    off = torch.from_numpy(off_h).to(dev)
    if timing is not None:
        timing["count"] = timing.get("count", 0.0) + time.perf_counter() - t0
        timing["count_kernel"] = timing.get("count_kernel", 0.0) + ev[0].elapsed_time(ev[1]) / 1e3
    os.makedirs(log_dir, exist_ok=True)
    paths = [os.path.join(log_dir, f"{int(seeds[g][0])}_{int(seeds[g][1])}_{split_names[g % len(split_names)]}.json.gz")
             for g in range(n)]
    pending = []  # (futures, pinned buffer) of the chunk before: at most two chunks' text is held at once
    g0 = 0
    while g0 < n:
        g1 = g0 + 1
        while g1 < n and off_h[g1 + 1] - off_h[g0] <= CHUNK_BYTES:
            g1 += 1
        size = int(off_h[g1] - off_h[g0])
        t1 = time.perf_counter()
        out = torch.empty(max(size, 1), dtype=torch.uint8, device=dev)
        if ev:
            ev[0].record(stream)
        _lib.check(L.mjx_mjai_render_fill_dev(*common, C.c_void_p(status.data_ptr()), C.c_void_p(off.data_ptr()), g0, g1,
                                              C.c_void_p(out.data_ptr()), size, sp), "mjx_mjai_render_fill_dev")
        if ev:
            ev[1].record(stream)
        host = torch.empty(max(size, 1), dtype=torch.uint8, pin_memory=True)
        host.copy_(out, non_blocking=True)
        stream.synchronize()
        del out
        if timing is not None:
            timing["fill_d2h"] = timing.get("fill_d2h", 0.0) + time.perf_counter() - t1
            timing["fill_kernel"] = timing.get("fill_kernel", 0.0) + ev[0].elapsed_time(ev[1]) / 1e3
        if pending:
            for f in pending[0]:
                f.result()
        buf = memoryview(host.numpy())
        base = int(off_h[g0])
        futs = [pool.submit(_write_gz, paths[g], heads[g][0], buf[int(off_h[g]) - base:int(off_h[g + 1]) - base], heads[g][1])
                for g in range(g0, g1)]
        pending = [futs, host]
        g0 = g1
    t2 = time.perf_counter()
    if pending:
        for f in pending[0]:
            f.result()
    if timing is not None:
        timing["gzip_wait"] = timing.get("gzip_wait", 0.0) + time.perf_counter() - t2
    return paths
