"""Data-parallel policy-net training (mortal_b200.train under torch.distributed): the split BatchNorm entries of the C ABI against
the single-process entries (bit for bit at one rank) and against float64 BatchNorm + Mish over all ranks' rows; and, with two
gloo ranks sharing one GPU (tests/ddp_train_worker.py under torch.distributed.run on 127.0.0.1), first-step gradients against
float64 over the whole batch, 20 AdamW steps against one process with the ranks' states bitwise equal, and train() itself:
saves, shards, the test play and its Stat, the stop rule and the illegal-action error. The NCCL command line needs two GPUs."""
from __future__ import annotations

import json
import os
import signal
import socket
import subprocess
import sys

import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from test_gpu_train import STATE_KEYS, _toml, arena_logs, tiny_cfg  # noqa: E402,F401
from test_gpu_train_ops import bn_mish_ref, check, make_bn  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "ddp_train_worker.py")


# ---- the split BatchNorm entries, one process -----------------------------------------------------------------------------------

def rows_of(n, c, dtype, seed):
    """[n, C, 1, 1] channels-last activations (n rows), with a constant channel and a channel of mean 1e3 and std 0.1"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((n, c, 1, 1), generator=g, device="cuda") * 1.5 + 0.3
    x[:, 0] = 0.75
    x[:, 1] = 1e3 + 0.1 * torch.randn((n, 1, 1), generator=g, device="cuda")
    return x.to(dtype).contiguous(memory_format=torch.channels_last)


def bits(t):
    return t.contiguous().view({torch.float32: torch.int32, torch.float16: torch.int16, torch.float64: torch.int64}[t.dtype])


class Ranks:
    """the split entries for `world` simulated ranks in one process, each holding its own rows and its own BatchNorm copy"""

    def __init__(self, xs, bn, eps=1e-3, momentum=0.01):
        from mortal_b200 import train_ops as O

        self.O, self.L, self.xs, self.world = O, O.ranks_lib(), xs, len(xs)
        self.c = c = xs[0].shape[1]
        self.code = O._dtype_code(xs[0])
        self.bns = [(bn.weight.detach().clone(), bn.bias.detach().clone(), bn.running_mean.clone(), bn.running_var.clone())
                    for _ in xs]
        self.eps, self.momentum = eps, momentum
        self.scratch = [torch.empty(O._scratch_floats(x.shape[0], c), dtype=torch.float32, device="cuda") for x in xs]

    def forward(self):
        O, L, c, p, s = self.O, self.L, self.c, self.O._p, self.O._stream(self.xs[0])
        rows = []
        for r, x in enumerate(self.xs):
            buf = torch.zeros((self.world, 3, c), dtype=torch.float64, device="cuda")
            O._lib.check(L.mjx_train_bn_local_stats(self.code, p(x), x.shape[0], c, r, self.world, p(buf), p(self.scratch[r]), s))
            rows.append(buf)
        gathered = torch.stack(rows).sum(0)  # what the all_reduce SUM gives every rank
        self.saved, outs = [], []
        for r, (x, (w, b, rm, rv)) in enumerate(zip(self.xs, self.bns)):
            mean, invstd, out = torch.empty(2 * c, device="cuda"), torch.empty(c, device="cuda"), torch.empty_like(x)
            O._lib.check(L.mjx_train_bn_mish_fwd_ranks(self.code, p(x), p(w), p(b), p(rm), p(rv), p(mean), p(invstd), p(out),
                                                       x.shape[0], c, self.eps, self.momentum, p(gathered), self.world, s))
            self.saved.append((mean, invstd))
            outs.append(out)
        return outs

    def backward(self, douts):
        O, L, c, p, s = self.O, self.L, self.c, self.O._p, self.O._stream(self.xs[0])
        parts = []
        for r, (x, d, (w, b, _, _), (mean, invstd)) in enumerate(zip(self.xs, douts, self.bns, self.saved)):
            buf = torch.zeros((self.world, 2, c), dtype=torch.float64, device="cuda")
            O._lib.check(L.mjx_train_bn_bwd_local_sums(self.code, p(x), p(d), p(w), p(b), p(mean), p(invstd), x.shape[0], c, r,
                                                       self.world, p(buf), p(self.scratch[r]), s))
            parts.append(buf)
        gathered = torch.stack(parts).sum(0)
        total = sum(x.shape[0] for x in self.xs)
        res = []
        for r, (x, d, (w, b, _, _), (mean, invstd)) in enumerate(zip(self.xs, douts, self.bns, self.saved)):
            dx, dw, db = torch.empty_like(x), torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
            O._lib.check(L.mjx_train_bn_mish_bwd_ranks(self.code, p(x), p(d), p(w), p(b), p(mean), p(invstd), p(dx), p(dw), p(db),
                                                       x.shape[0], c, p(gathered), r, self.world, total, p(self.scratch[r]), s))
            res.append((dx, dw, db))
        return res


def single(x, bn, dout, eps=1e-3, momentum=0.01):
    """mjx_train_bn_mish_fwd / _bwd in training mode -> (out, mean, invstd, running_mean, running_var, dx, dgamma, dbeta)"""
    from mortal_b200 import _lib, train_ops as O

    L, p, s, c, n = _lib.load(), O._p, O._stream(x), x.shape[1], x.shape[0]
    w, b, rm, rv = bn.weight.detach().clone(), bn.bias.detach().clone(), bn.running_mean.clone(), bn.running_var.clone()
    scratch = torch.empty(O._scratch_floats(n, c), dtype=torch.float32, device="cuda")
    mean, invstd, out = torch.empty(2 * c, device="cuda"), torch.empty(c, device="cuda"), torch.empty_like(x)
    code = O._dtype_code(x)
    O._lib.check(L.mjx_train_bn_mish_fwd(code, p(x), p(w), p(b), p(rm), p(rv), p(mean), p(invstd), p(out), n, c, eps, momentum, 1,
                                         p(scratch), s))
    dx, dw, db = torch.empty_like(x), torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    O._lib.check(L.mjx_train_bn_mish_bwd(code, p(x), p(dout), p(w), p(b), p(mean), p(invstd), p(dx), p(dw), p(db), n, c, 1, p(scratch),
                                         s))
    return out, mean, invstd, rm, rv, dx, dw, db


@pytest.mark.parametrize("n", [2, 33, 512 * 34])
@pytest.mark.parametrize("c", [32, 192])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_one_rank_split_entries_equal_the_single_entries(n, c, dtype):
    x = rows_of(n, c, dtype, seed=n + c)
    dout = rows_of(n, c, dtype, seed=n + c + 1) * 0.01
    bn = make_bn(c, seed=c)
    ref = single(x, bn, dout)
    R = Ranks([x], bn)
    out, = R.forward()
    (dx, dw, db), = R.backward([dout])
    (mean, invstd), (_, _, rm, rv) = R.saved[0], R.bns[0]
    for name, got, want in zip(("out", "save_mean", "save_invstd", "running_mean", "running_var", "dx", "dgamma", "dbeta"),
                               (out, mean, invstd, rm, rv, dx, dw, db), ref):
        assert torch.equal(bits(got), bits(want)), name


@pytest.mark.parametrize("shards", [(17, 5), (9, 9), (7, 7, 2), (1, 4, 11)])
@pytest.mark.parametrize("c", [32, 192])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_ranks_against_float64_over_all_rows(shards, c, dtype):
    from test_gpu_train_ops import activations

    xs = [activations(b, c, dtype, seed=100 * r + b) for r, b in enumerate(shards)]  # [B_r, C, 1, 34]
    douts = [activations(b, c, dtype, seed=100 * r + b + 7) * 0.1 for r, b in enumerate(shards)]
    for d in douts:
        d[:, 1] = 0.05
    x, dout = torch.cat(xs), torch.cat(douts)
    bn = make_bn(c, seed=c)
    ref = bn_mish_ref(x, bn, True, dout)
    tor = bn_mish_ref(x, bn, True, dout, dtype64=dtype, amp=dtype == torch.float16)
    flat = lambda t: t.permute(0, 3, 2, 1).reshape(-1, t.shape[1], 1, 1).contiguous(memory_format=torch.channels_last)  # noqa: E731
    R = Ranks([flat(t) for t in xs], bn)
    outs = R.forward()
    back = R.backward([flat(t) for t in douts])
    for r in range(1, len(shards)):  # every rank computed the same statistics
        for a, b in zip(R.saved[r] + R.bns[r][2:], R.saved[0] + R.bns[0][2:]):
            assert torch.equal(bits(a), bits(b))
    unflat = lambda t, b: t.reshape(b, 34, c).permute(0, 2, 1).unsqueeze(2)  # noqa: E731
    out = torch.cat([unflat(o, b) for o, b in zip(outs, shards)])
    dx = torch.cat([unflat(g[0], b) for g, b in zip(back, shards)])
    dw, db = sum(g[1] for g in back), sum(g[2] for g in back)  # what a gradient all-reduce SUM gives
    for name, i, got in (("out", 0, out), ("dx", 1, dx), ("dgamma", 2, dw), ("dbeta", 3, db), ("running_mean", 4, R.bns[0][2]),
                         ("running_var", 5, R.bns[0][3])):
        check(name, got, ref[i], tor[i], dtype)


def test_split_entries_reject_bad_ranks():
    from mortal_b200 import _lib, train_ops as O

    L, p = O.ranks_lib(), O._p
    x = rows_of(8, 32, torch.float32, seed=1)
    buf = torch.zeros((2, 3, 32), dtype=torch.float64, device="cuda")
    scratch = torch.empty(O._scratch_floats(8, 32), dtype=torch.float32, device="cuda")
    for rank, world in ((2, 2), (-1, 2), (0, 0)):
        assert L.mjx_train_bn_local_stats(0, p(x), 8, 32, rank, world, p(buf), p(scratch), O._stream(x)) != 0
    f = torch.empty(64, device="cuda")
    assert L.mjx_train_bn_mish_bwd_ranks(0, p(x), p(x), p(f), p(f), p(f), p(f), p(x), p(f), p(f), 8, 32, p(buf), 0, 2, 7,
                                         p(scratch), O._stream(x)) != 0  # total_rows < rows


# ---- two ranks ------------------------------------------------------------------------------------------------------------------

def free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def torchrun(args, cwd, timeout, nproc=2, module=None):
    """torch.distributed.run on 127.0.0.1; on timeout the whole process group is killed, so no rank outlives the test"""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port())] + (["-m", module] if module else []) + args
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", PYTHONPATH=ROOT, OMP_NUM_THREADS="1")
    p = subprocess.Popen(cmd, cwd=cwd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, start_new_session=True)
    try:
        out, _ = p.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        os.killpg(p.pid, signal.SIGKILL)
        out, _ = p.communicate()
        pytest.fail(f"timed out after {timeout} s:\n{out[-4000:]}")
    return p.returncode, out


def run_worker(tmp_path, mode, timeout=900, **args):
    out = tmp_path / f"out_{mode}"
    out.mkdir(exist_ok=True)
    (tmp_path / f"{mode}.json").write_text(json.dumps({"out": str(out), **args}))
    rc, log = torchrun([WORKER, ROOT, mode, str(tmp_path / f"{mode}.json")], cwd=tmp_path, timeout=timeout)
    assert rc == 0, log[-6000:]
    return [json.loads((out / f"rank{r}.json").read_text()) for r in range(2)]


def test_two_ranks_first_step_gradients_against_float64(tmp_path):
    res = run_worker(tmp_path, "grads")
    assert all(len(r["checked"]) == 6 for r in res)


def test_two_ranks_adamw_steps_agree_with_one_process(tmp_path):
    res = run_worker(tmp_path, "adamw")
    assert res[0]["losses"] == res[1]["losses"]


def test_two_rank_train(arena_logs, tmp_path):
    from mortal_b200.model import load_mortal
    from mortal_b200.player import TestPlayer
    from mortal_b200.stat import COUNTERS, Stat
    from mortal_b200.train import train

    cfg = tiny_cfg(tmp_path, "ddp", arena_logs / "logs")
    res = run_worker(tmp_path, "train", cfg=cfg, steps=4)
    assert [r["total"] for r in res] == [4, 4] and all("error" not in r for r in res)
    state_file = cfg["control"]["state_file"]
    assert res[1]["saves"] == [] and state_file in res[0]["saves"]
    state = torch.load(state_file, weights_only=True)
    assert set(state) == STATE_KEYS and state["steps"] == 4
    # the shards: disjoint, covering the index's list
    files = torch.load(cfg["dataset"]["file_index"], weights_only=True)["file_list"]
    a, b = set(res[0]["shard"]), set(res[1]["shard"])
    assert not a & b and a | b == set(files) and len(res[0]["shard"]) == len(res[1]["shard"]) == len(files) // 2
    # the test play: one process's file names, and the Stat is the sum of the ranks' own
    names = sorted(os.listdir(cfg["test_play"]["log_dir"]))
    assert len(names) == 8
    own = [r["local_stats"] for r in res]
    assert all(len(o) == 1 for o in own) and res[0]["test_stats"] == res[1]["test_stats"]
    assert res[0]["test_stats"][0] == [x + y for x, y in zip(own[0][0], own[1][0])]
    from_dir = Stat.from_dir(cfg["test_play"]["log_dir"], "mortal", disable_progress_bar=True)
    assert [getattr(from_dir, c) for c in COUNTERS] == res[0]["test_stats"][0]
    brain, dqn = load_mortal(state)  # strict
    single_dir = tmp_path / "single_play"
    tp = TestPlayer({**cfg, "test_play": {**cfg["test_play"], "log_dir": str(single_dir)}})
    tp.test_play(2, brain.cuda(), dqn.cuda(), torch.device("cuda", 0))
    assert sorted(os.listdir(single_dir)) == names
    # the state resumes in one process
    *_, steps = train(cfg, steps=2)
    assert steps == 6 and torch.load(state_file, weights_only=True)["steps"] == 6


def test_two_rank_train_stops_when_the_smaller_shard_runs_out(arena_logs, tmp_path):
    cfg = tiny_cfg(tmp_path, "stop", arena_logs / "logs")
    logs = sorted(os.listdir(arena_logs / "logs"))
    cfg["dataset"]["globs"] = [str(arena_logs / "logs" / f) for f in logs[:3]]  # shards of 2 and 1 files
    cfg["control"].update(save_every=1000, test_every=1000)
    res = run_worker(tmp_path, "train", cfg=cfg, steps=None)
    steps = res[0]["total"]
    assert res[1]["total"] == steps > 0
    assert [len(r["shard"]) for r in res] == [2, 1]
    assert res[1]["exhausted"] and res[1]["full_batches"] == steps  # the one-file shard ran out
    assert not res[0]["exhausted"] and res[0]["full_batches"] == steps + 1  # its next batch was never trained on


def test_two_rank_illegal_action_raises_on_both_ranks(arena_logs, tmp_path):
    cfg = tiny_cfg(tmp_path, "bad", arena_logs / "logs")
    res = run_worker(tmp_path, "train", cfg=cfg, steps=2, corrupt_rank=1)
    assert "step 1" in res[0]["error"] and res[0]["error"] == res[1]["error"]
    assert not os.path.exists(cfg["control"]["state_file"])


def test_command_line_nccl(arena_logs, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cfg = tiny_cfg(tmp_path, "cli", arena_logs / "logs")
    cfg["control"]["test_every"] = 1000
    (tmp_path / "tiny.toml").write_text(_toml(cfg))
    rc, log = torchrun([str(tmp_path / "tiny.toml")], cwd=tmp_path, timeout=900, module="mortal_b200.train")
    assert rc == 0, log[-6000:]
    state = torch.load(cfg["control"]["state_file"], weights_only=True)
    assert set(state) == STATE_KEYS and state["steps"] >= 2 and state["steps"] % 2 == 0
