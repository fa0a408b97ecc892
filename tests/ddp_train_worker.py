"""One rank of the data-parallel training checks in tests/test_gpu_train_ddp.py, started by torch.distributed.run over gloo (two
ranks may share one GPU): `python ddp_train_worker.py ROOT MODE ARGS.json`. Each rank writes its findings to
ARGS["out"]/rank{R}.json; an assertion failure exits non-zero.

- grads: the first-step gradients of every parameter and the BatchNorm running statistics, each rank on half of a batch, after
  the gradient all-reduce, against float64 torch over the whole batch (test_first_step_gradients_against_float64's bound, with
  4 eps more per rank for the per-rank rounding before the all-reduce).
- adamw: 20 AdamW + GradScaler steps on two ranks against one process at the same global batch; after every step the ranks'
  parameters, buffers, optimizer and scaler state are compared bit for bit.
- train: mortal_b200.train.train(ARGS["cfg"], ARGS["steps"]) with its saves, shards, test-play Stats and errors recorded.
"""
from __future__ import annotations

import copy
import json
import os
import sys

sys.path.insert(0, sys.argv[1])
sys.path.insert(0, os.path.join(sys.argv[1], "tests"))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

MODE, ARGS = sys.argv[2], json.load(open(sys.argv[3]))


def all_reduce_mean_grads(params, world):
    """what mortal_b200.train averages once per optimizer step"""
    grads = [p.grad for p in params if p.grad is not None]
    flat = torch.cat([g.reshape(-1) for g in grads])
    dist.all_reduce(flat)
    flat /= world
    o = 0
    for g in grads:
        g.copy_(flat[o:o + g.numel()].view_as(g))
        o += g.numel()


def fused_loss(brain, dqn, aux, bt, group):
    from mortal_b200 import train_ops
    from test_gpu_train import GAMMA, MIN_Q, NEXT_RANK

    obs, actions, masks, steps_to_done, rewards, ranks = bt
    phi = brain.forward_train(obs, group=group)
    v, a = dqn.heads(phi)
    dqn_loss, cql_loss, nr_loss, *_ = train_ops.dqn_losses(v, a, aux(phi)[0], masks, actions, steps_to_done, rewards, ranks, GAMMA)
    return dqn_loss + cql_loss * MIN_Q + nr_loss * NEXT_RANK


def half(bt, rank, world):
    n = bt[0].shape[0] // world
    return tuple(t[rank * n:(rank + 1) * n] for t in bt)


def check_grads(rank, world):
    import test_gpu_train as G

    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    checked = []
    for version, c, n, b in ((4, 192, 40, 32), (2, 32, 2, 16), (3, 32, 2, 16)):
        for dtype in (torch.float32, torch.float16):
            base = G.models(version, c, n, seed=version)  # the same seed on every rank
            bt = G.batch(version, b, seed=version + 10, jitter=True)
            amp = dtype == torch.float16
            scale = 1024.0 if amp else 1.0
            fus = [copy.deepcopy(m).train() for m in base]
            with torch.autocast("cuda", enabled=amp):
                lf = fused_loss(*fus, half(bt, rank, world), dist.group.WORLD)
            params = [p for m in fus for p in m.parameters()]
            (lf * scale).backward()
            all_reduce_mean_grads(params, world)
            gf = [p.grad.double() / scale for p in params]
            ref64 = [copy.deepcopy(m).double().train() for m in base]
            g64 = G.grads(ref64, G.torch_loss(*ref64, bt, torch.float64))
            tor = [copy.deepcopy(m).train() for m in base]
            with torch.autocast("cuda", enabled=amp):
                lt = G.torch_loss(*tor, bt)
            gt = G.grads(tor, lt, scale)
            names = [n_ for m in base for n_, _ in m.named_parameters()]
            eps = torch.finfo(dtype).eps
            # one process's bound plus 4 eps per rank: each rank's gradient is rounded to float32 at its own half batch before
            # the all-reduce adds them and the sum is rounded again (a scalar such as the value head's bias, a sum of cancelling
            # per-row terms, measured 1.3 eps over 2 e_torch + 8 eps at two ranks)
            slack = 8 + 4 * world
            for name, a, t, r in zip(names, gf, gt, g64):
                den = r.abs().max().item()
                e, et = ((a - r).abs().max().item() / den, (t - r).abs().max().item() / den) if den > 0 else (0.0, 0.0)
                assert e <= 2 * et + slack * eps, f"v{version} {dtype} {name}: e {e:.3e} > 2 * torch e {et:.3e} + {slack} eps"
            for mt, mf, m64 in zip(tor[0].modules(), fus[0].modules(), ref64[0].modules()):
                if isinstance(mt, torch.nn.BatchNorm1d):
                    assert int(mf.num_batches_tracked) == 1
                    for k in ("running_mean", "running_var"):
                        r, t, f = getattr(m64, k), getattr(mt, k).double(), getattr(mf, k).double()
                        den = r.abs().max().item()
                        assert (f - r).abs().max().item() / den <= 2 * (t - r).abs().max().item() / den + 8 * eps, k
            checked.append(f"v{version}-{c}x{n}-{dtype}")
    return {"checked": checked}


def state_bytes(ms, opt, scaler):
    """every parameter, buffer, optimizer and scaler state tensor as one CPU byte string"""
    ts = [t for m in ms for t in m.state_dict().values()]
    for s in opt.state.values():
        ts += [v if torch.is_tensor(v) else torch.tensor(v) for _, v in sorted(s.items())]
    ts += [scaler._scale, scaler._growth_tracker]
    return torch.cat([t.detach().reshape(-1).cpu().contiguous().view(torch.uint8) for t in ts])


def check_adamw(rank, world):
    import test_gpu_train as G

    base = G.models(4, 64, 6, seed=7)
    arms = {}
    for arm in ("one", "ranks"):
        ms = [copy.deepcopy(m).train() for m in base]
        params = [p for m in ms for p in m.parameters()]
        opt = torch.optim.AdamW(params, lr=1e-4)
        scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 10)
        losses = []
        for step in range(20):
            opt.zero_grad(set_to_none=True)
            bt = G.batch(4, 128, seed=100 + step % 5)
            if arm == "one":
                loss = fused_loss(*ms, bt, None)
            else:
                loss = fused_loss(*ms, half(bt, rank, world), dist.group.WORLD)
            scaler.scale(loss).backward()
            if arm == "ranks":
                all_reduce_mean_grads(params, world)
                loss = loss.detach().clone()
                dist.all_reduce(loss)
                loss /= world
            scaler.step(opt)
            scaler.update()
            losses.append(loss.item())
            if arm == "ranks":
                mine = state_bytes(ms, opt, scaler)
                got = [torch.empty_like(mine) for _ in range(world)]
                dist.all_gather(got, mine)
                assert all(torch.equal(g, got[0]) for g in got), f"step {step}: the ranks' states differ"
        arms[arm] = (ms, losses)
    (m1, l1), (mr, lr) = arms["one"], arms["ranks"]
    for step, (a, b) in enumerate(zip(lr, l1)):
        assert abs(a - b) <= 1e-3 * abs(b), f"step {step}: two-rank loss {a} vs one process {b}"
    for b1, br in zip(m1[0].modules(), mr[0].modules()):
        if isinstance(b1, torch.nn.BatchNorm1d):
            assert int(b1.num_batches_tracked) == int(br.num_batches_tracked) == 20
            torch.testing.assert_close(br.running_mean, b1.running_mean, rtol=1e-3, atol=1e-4)
            torch.testing.assert_close(br.running_var, b1.running_var, rtol=1e-3, atol=1e-4)
    return {"losses": lr}


def run_train(rank, world):
    from mortal_b200 import player, train as T
    from mortal_b200.stat import COUNTERS

    rec = {"saves": [], "shard": None, "full_batches": 0, "exhausted": False, "local_stats": [], "test_stats": []}
    save = torch.save

    def recording_save(obj, f, *a, **k):
        rec["saves"].append(str(f))
        return save(obj, f, *a, **k)

    torch.save = recording_save
    corrupt = ARGS.get("corrupt_rank") == rank

    class Recording(T.FileDatasetsIter):
        def __init__(self, version, file_list, *a, **k):
            rec["shard"] = list(file_list)
            super().__init__(version, file_list, *a, **k)

        def __iter__(self):
            for i, (obs, actions, masks, *rest) in enumerate(super().__iter__()):
                if obs.shape[0] != self.batch_size:
                    break
                if corrupt and i == 0:
                    masks = masks.clone()
                    masks[0, actions[0]] = False
                rec["full_batches"] += 1
                yield (obs, actions, masks, *rest)
            rec["exhausted"] = True

    T.FileDatasetsIter = Recording
    from_games, test_play = player.Stat.from_games, player.TestPlayer.test_play

    def recording_from_games(*a, **k):
        st = from_games(*a, **k)
        rec["local_stats"].append([getattr(st, c) for c in COUNTERS])
        return st

    def recording_test_play(self, *a, **k):
        st = test_play(self, *a, **k)
        rec["test_stats"].append([getattr(st, c) for c in COUNTERS])
        return st

    player.Stat.from_games = staticmethod(recording_from_games)
    player.TestPlayer.test_play = recording_test_play
    try:
        *_, total = T.train(ARGS["cfg"], steps=ARGS.get("steps"))
        rec["total"] = total
    except ValueError as e:
        rec["error"] = str(e)
    return rec


def main():
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    torch.cuda.set_device(0)
    out = {"grads": check_grads, "adamw": check_adamw, "train": run_train}[MODE](rank, world)
    with open(os.path.join(ARGS["out"], f"rank{rank}.json"), "w") as f:
        json.dump(out, f)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
