"""GRP training on the device (csrc/mjx_grp_train.cuh, mortal_b200.grp_train, mortal_b200.train_grp): grp_loss against a
torch-CPU float64 restatement of train_grp.py's step at every supported shape class, bit-identical repeats and gradient
accumulation, GrpFileDatasetsIter against the restated reference iterator + DataLoader on arena logs, 200 AdamW steps against a
reference loop with torch's float64 GRU, the train() entry point (state file, strict loads both ways, resume), and rejections."""
import os
import random

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import grp_train_lib as T  # noqa: E402
from test_gpu_gameplay_decode import _Eng  # noqa: E402

LENGTHS = (1, 2, 8, 20, 64)


def device_grp(ref):
    """a mortal_b200.model.GRP on cuda:0 holding `ref`'s weights"""
    from mortal_b200.model import GRP

    g = GRP(ref.rnn.hidden_size, ref.rnn.num_layers)
    g.load_state_dict(ref.state_dict())
    return g.cuda()


def host_batch(feats, game, length, rank):
    from mortal_b200.grp_train import make_batch

    return make_batch(np.concatenate(feats), [len(f) for f in feats], game, length, rank)


@pytest.mark.parametrize("shape", [(64, 2), (32, 1), (96, 3), (256, 4), (1, 1)], ids=lambda p: f"H{p[0]}xL{p[1]}")
def test_grp_loss_matches_reference(shape):
    from mortal_b200.grp_train import grp_loss

    ref = T.random_grp(*shape, 500 + shape[0])
    dev = device_grp(ref)
    rng = np.random.default_rng(shape[0] + shape[1])
    feats = [T.random_feature(n, rng) for n in LENGTHS]
    ranks = np.array([rng.permutation(4) for _ in feats])
    random_game = rng.integers(0, len(LENGTHS), size=512)
    cases = [([0], [1]), ([4], [64]), ([3] * 20, np.arange(1, 21)), ([3, 3, 4, 4, 3], [5, 5, 64, 64, 20]),
             (random_game, [int(rng.integers(1, LENGTHS[g] + 1)) for g in random_game])]
    err = 0.0
    for game, length in cases:
        game, length = np.asarray(game), np.asarray(length)
        rank = ranks[game].copy()
        rank[0] = [0, 0, 1, 2]  # no permutation: label 0
        batch = host_batch(feats, game, length, rank)
        dev.zero_grad(set_to_none=True)
        loss, acc = grp_loss(dev, batch)
        assert loss.is_cuda and loss.dtype == torch.float64 and loss.dim() == 0 and acc.dim() == 0
        want_loss, want_acc = T.ref_step(ref, [torch.as_tensor(feats[g][:n]) for g, n in zip(game, length)], rank)
        assert abs(loss.item() - want_loss) <= 1e-12 * abs(want_loss)
        assert acc.item() == want_acc
        for p, r in zip(dev.parameters(), ref.parameters()):
            e = (p.grad.cpu() - r.grad).abs().max().item() / max(r.grad.abs().max().item(), 1e-300)
            err = max(err, e)
        # forward only: the same loss, no gradient touched
        dev.zero_grad(set_to_none=True)
        loss2, acc2 = grp_loss(dev, batch, backward=False)
        assert torch.equal(loss2, loss) and torch.equal(acc2, acc)
        assert all(p.grad is None for p in dev.parameters())
    print(f"H={shape[0]} layers={shape[1]}: max relative gradient error {err:.2e}")
    assert err <= 1e-12


def test_repeats_are_bit_identical_and_accumulate():
    from mortal_b200.grp_train import grp_loss

    dev = device_grp(T.random_grp(64, 2, 9))
    rng = np.random.default_rng(3)
    feats = [T.random_feature(n, rng) for n in LENGTHS]
    game = rng.integers(0, len(LENGTHS), size=512)
    length = [int(rng.integers(1, LENGTHS[g] + 1)) for g in game]
    batch = host_batch(feats, game, length, [rng.permutation(4) for _ in game])
    first = grp_loss(dev, batch)
    g1 = [p.grad.clone() for p in dev.parameters()]
    dev.zero_grad(set_to_none=True)
    second = grp_loss(dev, batch)
    assert torch.equal(first[0], second[0]) and torch.equal(first[1], second[1])
    assert all(torch.equal(p.grad, g) for p, g in zip(dev.parameters(), g1))
    grp_loss(dev, batch)  # adds to the existing .grad
    assert all(torch.equal(p.grad, g + g) for p, g in zip(dev.parameters(), g1))


@pytest.fixture(scope="module")
def arena_files(tmp_path_factory):
    from mortal_b200.libriichi.arena import OneVsThree

    d = tmp_path_factory.mktemp("arena_grp_train")
    OneVsThree(disable_progress_bar=True, log_dir=str(d)).py_vs_py(_Eng("alpha", 2.0), _Eng("beta", 0.5), (95000, 41), 16)
    files = sorted(os.path.join(d, f) for f in os.listdir(d))
    assert len(files) == 64
    return files


def ref_load(chunk):
    from mortal_b200.dataset import Grp

    return [(g.take_feature(), g.take_rank_by_player()) for g in Grp.load_gz_log_files(chunk)]


def prefixes(batch):
    feat, off = batch.feat.cpu(), batch.game_off.cpu().long()
    return [feat[off[g]:off[g] + n] for g, n in zip(batch.game.cpu().long().tolist(), batch.length.cpu().long().tolist())]


@pytest.mark.parametrize("cycle,batch_size,file_batch_size,n_batches", [(False, 100, 10, None), (True, 700, 3, 12),
                                                                         (True, 64, 50, 40)])
def test_iterator_matches_reference(arena_files, cycle, batch_size, file_batch_size, n_batches):
    from mortal_b200.grp_train import GrpFileDatasetsIter

    random.seed(77)
    want = T.ref_batches(T.RefGrpFileDatasetsIter(list(arena_files), ref_load, file_batch_size, cycle), batch_size, n_batches)
    state = random.getstate()
    random.seed(77)
    got = []
    for b in GrpFileDatasetsIter(list(arena_files), file_batch_size, cycle, batch_size=batch_size):
        got.append(b)
        if n_batches is not None and len(got) == n_batches:
            break
    assert random.getstate() == state
    assert len(got) == len(want) and len(want) >= (n_batches or 2)
    for b, w in zip(got, want):
        assert b.feat.is_cuda and b.rank_by_player.is_cuda and b.rank_by_player.dtype == torch.int64
        ps = prefixes(b)
        assert len(ps) == len(w)
        assert all(torch.equal(p, x) for p, (x, _) in zip(ps, w))
        assert b.rank_by_player.cpu().tolist() == [list(r) for _, r in w]


def test_training_matches_reference_loop(arena_files):
    from torch.nn import functional as F
    from torch.nn.utils.rnn import pack_padded_sequence, pad_sequence

    from mortal_b200.grp_train import GrpFileDatasetsIter, grp_loss

    steps, batch_size, lr = 200, 256, 1e-3
    random.seed(2024)
    ref_stream = T.ref_batches(T.RefGrpFileDatasetsIter(list(arena_files), ref_load, 50, True), batch_size, steps)
    random.seed(2024)
    it = iter(GrpFileDatasetsIter(list(arena_files), 50, True, batch_size=batch_size))
    dev_stream = [next(it) for _ in range(steps)]

    init = T.random_grp(64, 2, 123)
    ref = T.RefGRP(64, 2).cuda()
    ref.load_state_dict(init.state_dict())
    dev = device_grp(init)
    opt_r = torch.optim.AdamW(ref.parameters(), lr=lr)
    opt_d = torch.optim.AdamW(dev.parameters(), lr=lr)
    perms = ref.perms
    worst = 0.0
    for s in range(steps):
        inputs = [x for x, _ in ref_stream[s]]
        rank = torch.tensor([r for _, r in ref_stream[s]], dtype=torch.int64).cuda()
        packed = pack_padded_sequence(pad_sequence(inputs, batch_first=True), torch.tensor([len(x) for x in inputs]),
                                      batch_first=True, enforce_sorted=False).to("cuda")
        _, state = ref.rnn(packed)
        logits = ref.fc(state.transpose(0, 1).flatten(1))
        mappings = (perms.expand(len(rank), -1, -1).transpose(0, 1) == rank).all(-1).nonzero()
        labels = torch.zeros(len(rank), dtype=torch.int64, device="cuda")
        labels[mappings[:, 1]] = mappings[:, 0]
        loss_r = F.cross_entropy(logits, labels)
        opt_r.zero_grad(set_to_none=True)
        loss_r.backward()
        opt_r.step()

        opt_d.zero_grad(set_to_none=True)
        loss_d, _ = grp_loss(dev, dev_stream[s])
        opt_d.step()
        rel = abs(loss_d.item() - loss_r.item()) / abs(loss_r.item())
        worst = max(worst, rel)
        assert rel <= 1e-10, (s, loss_d.item(), loss_r.item())
    perr = max((p - q).abs().max().item() for p, q in zip(dev.parameters(), ref.parameters()))
    moved = max((p.cpu() - q).abs().max().item() for p, q in zip(dev.parameters(), init.parameters()))
    print(f"{steps} AdamW steps: max relative loss gap {worst:.2e}, max |param gap| {perr:.2e}, max weight change {moved:.2e}")
    assert perr <= 1e-9 and moved > 1e-2


def tiny_cfg(d, files, name):
    return {"state_file": os.path.join(d, f"{name}.pth"), "network": {"hidden_size": 16, "num_layers": 2},
            "control": {"device": "cuda:0", "enable_cudnn_benchmark": False, "tensorboard_dir": os.path.join(d, "tb"),
                        "batch_size": 0, "save_every": 2, "val_steps": 1},
            "dataset": {"train_globs": [os.path.join(files, "**", "*.json.gz")], "val_globs": [os.path.join(files, "*.json.gz")],
                        "file_index": os.path.join(d, f"{name}_index.pth"), "file_batch_size": 100},
            "optim": {"lr": 1e-3}}


def test_train_entry_point_saves_and_resumes(arena_files, tmp_path):
    from mortal_b200.dataset import Grp
    from mortal_b200.train_grp import train

    files = arena_files[:1]
    src = tmp_path / "logs"
    (src / "sub").mkdir(parents=True)
    os.symlink(files[0], src / "sub" / os.path.basename(files[0]))  # one level down: the globs are recursive
    n = sum(len(g.take_feature()) for g in Grp.load_gz_log_files(files))
    # one file and one batch per cycle (batch_size = every prefix of the file): the fresh iterators of a resumed call then draw
    # what the uninterrupted run draws (with more files, the reference's in-place shuffle of the file list would differ), so a
    # resumed run must reproduce the uninterrupted one exactly
    cfg_a, cfg_b = tiny_cfg(tmp_path, src, "a"), tiny_cfg(tmp_path, src, "b")
    cfg_b["dataset"]["val_globs"] = cfg_a["dataset"]["val_globs"] = cfg_a["dataset"]["train_globs"]
    for c in (cfg_a, cfg_b):
        c["control"]["batch_size"] = n
    torch.manual_seed(0)
    random.seed(0)
    train(cfg_a, steps=4)
    state = torch.load(cfg_a["state_file"], weights_only=True)
    assert state["steps"] == 4 and set(state) == {"model", "optimizer", "steps", "timestamp"}
    index = torch.load(cfg_a["dataset"]["file_index"], weights_only=True)
    assert index["train_file_list"] == index["val_file_list"] == [str(src / "sub" / os.path.basename(files[0]))]
    ref = T.RefGRP(16, 2)
    ref.load_state_dict(state["model"])  # strict
    opt = torch.optim.AdamW(ref.parameters())
    opt.load_state_dict(state["optimizer"])
    assert [k for k in state["model"]] == [k for k in T.RefGRP(16, 2).state_dict()]
    grp_a, _, steps_a = train(cfg_a, steps=4)  # resumes
    assert steps_a == 8 and torch.load(cfg_a["state_file"], weights_only=True)["steps"] == 8
    torch.manual_seed(0)
    random.seed(0)
    grp_b, _, steps_b = train(cfg_b, steps=8)
    assert steps_b == 8
    assert all(torch.equal(p, q) for p, q in zip(grp_a.parameters(), grp_b.parameters()))


def test_rejections():
    from mortal_b200.grp_train import grp_loss, make_batch
    from mortal_b200.model import GRP

    rng = np.random.default_rng(0)
    feats = [T.random_feature(n, rng) for n in (3, 5)]
    batch = host_batch(feats, [0, 1], [3, 5], [[0, 1, 2, 3]] * 2)
    for shape in ((257, 1), (8, 5)):
        with pytest.raises(ValueError):
            grp_loss(GRP(*shape).cuda(), batch)
    lens, feat = [3, 5], np.concatenate(feats)
    for game, length, rank in (([0, 2], [1, 1], [[0, 1, 2, 3]] * 2), ([0, 1], [4, 1], [[0, 1, 2, 3]] * 2),
                               ([0, 1], [0, 1], [[0, 1, 2, 3]] * 2), ([0, 1], [1, 1], [[0, 1, 2]] * 2), ([], [], [])):
        with pytest.raises(ValueError):
            make_batch(feat, lens, game, length, rank)
    with pytest.raises(ValueError):
        make_batch(feat[:7], lens, [0], [1], [[0, 1, 2, 3]])
    with pytest.raises(ValueError):
        grp_loss(GRP(16, 2).cuda(), batch._replace(rank_by_player=batch.rank_by_player[:1]))
