"""Online training with self-play actors beside the trainer: mortal/server.py's parameter server and buffer in the trainer process,
mortal/client.py's self-play loop in actor processes on any CUDA devices (`[online] actor_devices`), run by
`train.train_online` when that key is set.

    [online]
    actor_devices = ["cuda:1", "cuda:2"]   # one actor per entry; a device may repeat; the trainer's own device is allowed

Each actor is a process started with torch.multiprocessing's spawn method. It owns a Brain / DQN pair and a `player.TrainPlayer`
on its device (its `[baseline.train]` engine too, since the arena plays both engines on one GPU), and loops as mortal/client.py
does: fetch the latest parameters it may play, play one `train_play_games` session, submit the games. Games and parameters move
as CUDA tensors through CUDA IPC, never staged on the host or written to files:
- an actor sends its session's event words trimmed to the longest game, with the lengths, names, seeds, ranks and scores; the
  trainer copies them into its own buffer on its own device and acknowledges, and only then does the actor free them;
- the trainer publishes a versioned snapshot of the Brain and DQN state_dicts (BatchNorm buffers included) on its device, which
  actors copy into their own modules; the trainer's live modules are never played.

`Server` holds mortal/server.py's state and rules (server.py:51-118). A service thread per actor answers its requests while the
training loop runs; where the reference sleeps and retries (the client's 3 s, `drain`'s 5 s), the waiting side blocks on the
server's condition instead. The trainer publishes where mortal/train.py submits (idle at start, every `submit_every` steps, at a
save that is not on a submit, idle after each pass), and each round drains the buffer and runs one `SelfPlayDatasetsIter` pass
over the drained games in submission order, as the sequential loop trains on its own games.

Errors: an exception in an actor reaches the trainer with its traceback, and the trainer raises RuntimeError naming the actor's
index and device (an actor that exits without a report is named the same way). Whenever `train_concurrent` ends, normally or not,
it sets the stop event, discards the sessions in flight, joins every actor (terminating one that has not exited after
JOIN_TIMEOUT seconds) and returns only when no actor process is left.
"""
from __future__ import annotations

import copy
import logging
import queue
import secrets
import threading
import traceback
from dataclasses import dataclass

import numpy as np

JOIN_TIMEOUT = 10.0  # seconds an actor gets to finish its session after the stop event before it is terminated
_POLL = 0.5  # seconds between a service thread's liveness checks of its actor


@dataclass
class Submission:
    """one actor session's games as held by the trainer: the actor's index, the param version it played and the games
    (selfplay.SelfPlayGames on the trainer's device, words trimmed to the session's longest game)"""
    actor: int
    param_version: int
    games: object


class Server:
    """mortal/server.py's state, in the trainer process. Every method takes the one lock; `monitor(kind, **info)`, when given, is
    called under it for every publish ("publish": version, is_idle, snapshot), submission ("submit": actor, param_version, seeds,
    buffered, submission) and drain ("drain": submissions, param_version), so the events it sees are in the order the server
    applied them."""

    def __init__(self, capacity: int, force_sequential: bool, monitor=None):
        self.capacity, self.force_sequential, self.monitor = capacity, force_sequential, monitor
        self.cond = threading.Condition()
        self.snapshot = None
        self.param_version = self.idle_param_version = 0
        self.buffer, self.buffer_size = [], 0
        self.closed = False
        self.error = None

    def _event(self, kind, **info):
        if self.monitor is not None:
            self.monitor(kind, **info)

    def _get_param(self, client_version):
        """server.py:51-78"""
        if self.buffer_size >= self.capacity:
            return {"status": "samples overflow"}
        if self.snapshot is None:
            return {"status": "empty param"}
        if self.force_sequential and self.idle_param_version <= client_version:
            return {"status": "trainer is busy"}
        return {"status": "ok", "snapshot": self.snapshot, "param_version": self.param_version}

    def get_param(self, client_version):
        """the answer to an actor holding `client_version` (-1: none yet): {"status": "ok", "snapshot", "param_version"}, or
        {"status": "samples overflow" | "empty param" | "trainer is busy"}"""
        with self.cond:
            return self._get_param(client_version)

    def wait_param(self, client_version):
        """get_param, blocking until its status is "ok"; None once the server is closed"""
        with self.cond:
            while not self.closed:
                res = self._get_param(client_version)
                if res["status"] == "ok":
                    return res
                self.cond.wait()
            return None

    def submit_param(self, snapshot, is_idle: bool):
        """server.py:95-101: the new snapshot gets the next version, which is also the idle version when `is_idle`. RuntimeError
        when an actor has failed."""
        with self.cond:
            self._raise()
            self.snapshot = snapshot
            self.param_version += 1
            if is_idle:
                self.idle_param_version = self.param_version
            self._event("publish", version=self.param_version, is_idle=is_idle, snapshot=snapshot)
            self.cond.notify_all()
            return self.param_version

    def submit_replay(self, actor: int, param_version: int, games):
        """server.py:84-93: buffer one session's games (dropped once the server is closed)"""
        with self.cond:
            if self.closed:
                return
            sub = Submission(actor, param_version, games)
            self.buffer.append(sub)
            self.buffer_size += len(games)
            self._event("submit", actor=actor, param_version=param_version, seeds=list(games.seeds), buffered=self.buffer_size,
                        submission=sub)
            self.cond.notify_all()

    def drain(self, wait: bool = False):
        """server.py:103-118: every buffered submission, in submission order, when there is at least one game (with
        force_sequential, at least `capacity`); else [], or with `wait` block until there is. RuntimeError when an actor has
        failed, also while waiting."""
        with self.cond:
            while True:
                self._raise()
                if self.buffer_size > 0 and (not self.force_sequential or self.buffer_size >= self.capacity):
                    taken, self.buffer, self.buffer_size = self.buffer, [], 0
                    self._event("drain", submissions=list(taken), param_version=self.param_version)
                    self.cond.notify_all()
                    return taken
                if not wait or self.closed:
                    return []
                self.cond.wait()

    def fail(self, message: str):
        """an actor failed: the trainer's next publish or drain raises RuntimeError(message), and the server closes"""
        with self.cond:
            if self.error is None:
                self.error = message
            self.closed = True
            self.cond.notify_all()

    def close(self):
        """no more parameters are handed out and no more games are taken; every waiter wakes"""
        with self.cond:
            self.closed = True
            self.cond.notify_all()

    def _raise(self):
        if self.error is not None:
            raise RuntimeError(self.error)


def parse_actor_devices(devices):
    """`[online] actor_devices` -> list of torch.device; ValueError for an entry that is not a CUDA device"""
    import torch

    if not isinstance(devices, (list, tuple)):
        raise ValueError(f"[online] actor_devices must be a list of CUDA device strings, got {devices!r}")
    out = []
    for i, s in enumerate(devices):
        try:
            dev = torch.device(s) if isinstance(s, str) else None
        except RuntimeError:
            dev = None
        if dev is None or dev.type != "cuda":
            raise ValueError(f"[online] actor_devices[{i}] = {s!r} is not a CUDA device (expected e.g. \"cuda:1\")")
        out.append(torch.device("cuda", dev.index or 0))
    return out


# ---- actor process -----------------------------------------------------------------------------------------------------------
def _actor_main(idx, device, config, train_key, requests, replies, stop, log_level, cudnn_deterministic):
    """mortal/client.py:35-80 on `device`, talking to the trainer through `requests` / `replies`, with the trainer process's
    cudnn.deterministic (so a deterministic trainer plays as the sequential loop would in its own process)"""
    logging.basicConfig(level=log_level, format=f"%(asctime)s %(levelname)s actor {idx} ({device}): %(message)s")
    try:
        import torch
        import torch.multiprocessing  # noqa: F401  (registers the CUDA IPC reductions the queues pickle with)

        from .model import DQN, Brain
        from .player import TrainPlayer

        dev = torch.device(device)
        torch.cuda.set_device(dev)
        torch.backends.cudnn.deterministic = cudnn_deterministic
        cfg = copy.deepcopy(config)
        cfg["baseline"]["train"]["device"] = str(dev)  # the arena plays both engines on the actor's GPU
        version = cfg["control"]["version"]
        mortal = Brain(version=version, **cfg["resnet"]).to(dev).eval()
        dqn = DQN(version=version).to(dev)
        player = TrainPlayer(cfg)
        player.train_key = train_key
        pts = np.array([90, 45, 0, -135])
        history_window = cfg["online"]["history_window"]
        history = []
        param_version = -1
        while not stop.is_set():
            requests.put(("get_param", param_version))
            rsp = replies.get()
            if rsp is None:  # the trainer is stopping
                break
            snapshot, param_version = rsp
            mortal.load_state_dict(snapshot["mortal"])
            dqn.load_state_dict(snapshot["dqn"])
            torch.cuda.synchronize(dev)
            del rsp, snapshot  # the trainer's snapshot is released before the next request
            logging.info("param has been updated")

            rankings, games = player.train_play_games(mortal, dqn, dev)
            history.append(np.array(rankings))
            if len(history) > history_window:
                del history[0]
            total_r = np.sum(history, axis=0)
            logging.info(f"trainee rankings: {rankings} ({rankings @ np.arange(1, 5) / rankings.sum():.6}, "
                         f"{rankings @ pts / rankings.sum():.6}pt)")
            logging.info(f"last {len(history)} sessions: {total_r} ({total_r @ np.arange(1, 5) / total_r.sum():.6}, "
                         f"{total_r @ pts / total_r.sum():.6}pt)")
            if stop.is_set():
                break
            words, lens = games.words[:, :min(int(games.lens.max()), games.words.shape[1])].contiguous(), games.lens
            torch.cuda.synchronize(dev)
            requests.put(("submit", param_version, (words, lens, games.log_cap, games.names, games.seeds, games.ranks,
                                                    games.scores)))
            del games
            if replies.get() is None:  # the acknowledgement: the trainer holds its own copy, these tensors may go
                break
            del words, lens
            logging.info("games have been submitted")
    except KeyboardInterrupt:
        pass
    except BaseException:
        requests.put(("error", traceback.format_exc()))


# ---- trainer side --------------------------------------------------------------------------------------------------------------
class _Actor:
    """one actor process and the trainer thread that serves it"""

    def __init__(self, ctx, idx, device, config, train_key, server, trainer_device, stop):
        import torch

        self.idx, self.device, self.server, self.trainer_device = idx, device, server, trainer_device
        self.name = f"actor {idx} ({device})"
        self.requests, self.replies = ctx.Queue(), ctx.Queue()
        self.proc = ctx.Process(target=_actor_main, name=f"mortal-actor-{idx}", daemon=True,
                                args=(idx, str(device), config, train_key, self.requests, self.replies, stop,
                                      logging.getLogger().getEffectiveLevel(), torch.backends.cudnn.deterministic))
        self.thread = threading.Thread(target=self._serve, name=f"mortal-actor-{idx}-service", daemon=True)

    def start(self):
        self.proc.start()
        self.thread.start()

    def _serve(self):
        try:
            import torch

            self.stream = torch.cuda.Stream(self.trainer_device)
            while True:
                try:
                    msg = self.requests.get(timeout=_POLL)
                except queue.Empty:
                    if self.proc.exitcode is None:
                        continue
                    try:  # a message sent just before the exit is in the pipe by now
                        msg = self.requests.get_nowait()
                    except queue.Empty:
                        if not self.server.closed:
                            self.server.fail(f"{self.name} exited with code {self.proc.exitcode} without reporting an error")
                        return
                msg = list(msg)
                self._handle(msg)  # empties msg: no reference to the actor's tensors outlives their copy
        except BaseException:
            self.server.fail(f"the trainer's service thread of {self.name} failed:\n{traceback.format_exc()}")

    def _handle(self, msg):
        import torch

        from .selfplay import SelfPlayGames

        kind, args = msg[0], msg[1:]
        msg.clear()
        if kind == "get_param":
            res = self.server.wait_param(args[0])
            self.replies.put(None if res is None else (res["snapshot"], res["param_version"]))
        elif kind == "submit":
            param_version, (words, lens, log_cap, names, seeds, ranks, scores) = args
            del args
            games = None
            if not self.server.closed:
                with torch.cuda.stream(self.stream):  # off the training stream; _take makes that stream wait for it
                    games = SelfPlayGames(words.to(self.trainer_device, copy=True), lens.to(self.trainer_device, copy=True),
                                          log_cap, names, seeds, ranks, scores)
                self.stream.synchronize()
            del words, lens  # the actor's tensors are released before it may free them
            self.replies.put("ack")
            if games is not None:
                self.server.submit_replay(self.idx, param_version, games)
        elif kind == "error":
            self.server.fail(f"{self.name} failed:\n{args[0]}")
        else:
            raise ValueError(f"unknown request {kind!r} from {self.name}")


def _take(submissions, device):
    """the drained submissions' games as one selfplay.SelfPlayGames, in submission order, their trimmed words zero-padded back to
    the arena's log capacity (the words converter takes rows of at least that many words)"""
    import torch

    from .selfplay import SelfPlayGames

    cur = torch.cuda.current_stream(device)
    parts = [s.games for s in submissions]
    caps = {p.log_cap for p in parts}
    if len(caps) != 1:
        raise ValueError(f"the drained games' log capacities differ ({sorted(caps)})")
    log_cap = caps.pop()
    words = torch.zeros((sum(len(p) for p in parts), log_cap), dtype=torch.int64, device=device)
    row = 0
    for p in parts:
        p.words.record_stream(cur)  # copied on a service thread's stream, read (and freed) on this one
        p.lens.record_stream(cur)
        words[row:row + len(p), :p.words.shape[1]] = p.words
        row += len(p)
    return SelfPlayGames(words, torch.cat([p.lens for p in parts]), log_cap, [x for p in parts for x in p.names],
                         [x for p in parts for x in p.seeds], np.concatenate([p.ranks for p in parts]),
                         np.concatenate([p.scores for p in parts]))


def _snapshot(T):
    """the trainer's Brain and DQN state_dicts, BatchNorm buffers included, as fresh tensors on its device"""
    import torch

    snap = {name: {k: v.detach().clone() for k, v in m.state_dict().items()} for name, m in (("mortal", T.mortal), ("dqn", T.dqn))}
    torch.cuda.current_stream(T.device).synchronize()  # complete before any actor reads it
    return snap


def _shutdown(actors, server, stop):
    stop.set()
    server.close()
    for a in actors:
        if a.proc.pid is not None:
            a.replies.put(None)  # wakes an actor waiting for parameters or an acknowledgement
    for a in actors:
        if a.proc.pid is None:
            continue
        a.proc.join(JOIN_TIMEOUT)
        if a.proc.is_alive():
            logging.warning(f"{a.name} did not stop within {JOIN_TIMEOUT} s: terminating it")
            a.proc.terminate()
            a.proc.join()
    for a in actors:
        if a.thread.is_alive():
            a.thread.join()
        for q in (a.requests, a.replies):
            q.cancel_join_thread()
            q.close()


def train_concurrent(config, rounds=None, steps=None, monitor=None):
    """train_online with `[online] actor_devices` (module docstring): `rounds` bounds the call to that many drains trained on,
    `steps` to that many training steps. Returns (brain, dqn, aux_net, optimizer, total steps)."""
    import torch.multiprocessing as mp

    from .train import _load_grp, _train_pass, _Trainer, check_online_config

    check_online_config(config)
    devices = parse_actor_devices(config["online"]["actor_devices"])
    server_cfg = config["online"]["server"]
    server = Server(server_cfg["capacity"], server_cfg.get("force_sequential", False), monitor)
    T = _Trainer(config, online=True)
    grp = _load_grp(config)
    T.publish = lambda is_idle: server.submit_param(_snapshot(T), is_idle)
    keys = [secrets.randbits(64) for _ in devices]  # one train_key per actor, as each reference client draws its own
    ctx = mp.get_context("spawn")
    stop = ctx.Event()
    actors = [_Actor(ctx, i, d, config, k, server, T.device, stop) for i, (d, k) in enumerate(zip(devices, keys))]
    try:
        for a in actors:
            a.start()
        logging.info(f"{len(actors)} self-play actors on {', '.join(str(d) for d in devices)}")
        T.publish(True)  # mortal/train.py:129-131
        done = rounds_done = 0
        while (rounds is None or rounds_done < rounds) and (steps is None or done < steps):
            taken = server.drain(wait=True)
            if not taken:
                raise RuntimeError("the parameter server closed while the trainer was waiting for games")
            games = _take(taken, T.device)
            versions = [s.param_version for s in taken]
            logging.info(f"round {rounds_done + 1}: {len(games):,} games from {len(taken)} sessions (param versions "
                         f"{min(versions)}..{max(versions)}, latest {server.param_version}); total steps: {T.total:,} "
                         f"(~{(T.test_every - T.total % T.test_every) % T.test_every:,})")
            del taken
            done = _train_pass(T, config, grp, games, steps, done)
            del games
            rounds_done += 1
            T.publish(True)  # mortal/train.py:425-427
    finally:
        _shutdown(actors, server, stop)
        T.publish = None
    T.check_actions()
    return T.mortal, T.dqn, T.aux_net, T.optimizer, T.total
