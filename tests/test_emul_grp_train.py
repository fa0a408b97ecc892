"""The GRP training step (csrc/mjx_grp_train.cuh, host build) against a torch-CPU float64 restatement of train_grp.py's step
(pack_padded_sequence over every sample's prefix, forward_packed, get_label, F.cross_entropy, backward()): every gradient tensor
within 1e-12 of the reference relative to its largest |value|, the loss within 1e-12 relative, the accuracy exactly; a
forward-only call writes no gradient; bad arguments and bad samples give the documented codes."""
import numpy as np
import pytest
import torch

import grp_train_lib as T

LENGTHS = (1, 2, 8, 20, 64)
SHAPES = [(64, 2), (32, 1), (96, 3), (256, 4), (1, 1), (1, 3)]


@pytest.fixture(scope="module", params=SHAPES, ids=lambda p: f"H{p[0]}xL{p[1]}")
def net(request):
    hidden, layers = request.param
    grp = T.random_grp(hidden, layers, 300 + hidden + layers)
    rng = np.random.default_rng(hidden * 10 + layers)
    feats = [T.random_feature(n, rng) for n in LENGTHS]
    ranks = np.array([rng.permutation(4) for _ in feats])
    return grp, T.pack(grp), feats, ranks


def check(net, game, length, rank=None, grad=True):
    grp, (w, h, nl), feats, ranks = net
    game, length = np.asarray(game), np.asarray(length)
    rank = ranks[game] if rank is None else rank
    rc, loss, acc, g, status = T.run_emul(w, h, nl, feats, game, length, rank, grad=grad)
    assert rc == 0 and not status.any()
    inputs = [torch.as_tensor(feats[a][:b]) for a, b in zip(game, length)]
    want_loss, want_acc = T.ref_step(grp, inputs, rank, backward=grad)
    assert abs(loss - want_loss) <= 1e-12 * abs(want_loss), (loss, want_loss)
    assert acc == want_acc
    if not grad:
        assert np.isnan(g).all()
        return 0.0
    err = T.grad_err(g, grp)
    assert err <= 1e-12, err
    return err


def test_one_sample(net):
    for gi, n in enumerate(LENGTHS):
        check(net, [gi], [n])
        check(net, [gi], [1])


def test_every_prefix_of_one_game(net):
    for gi, n in enumerate(LENGTHS):
        check(net, [gi] * n, np.arange(1, n + 1))


def test_duplicated_samples(net):
    check(net, [3, 3, 3, 1, 1, 3], [5, 5, 20, 2, 2, 5])
    check(net, [4] * 4, [64] * 4)


def test_random_batches_of_512(net):
    rng = np.random.default_rng(11)
    game = rng.integers(0, len(LENGTHS), size=512)
    length = np.array([rng.integers(1, LENGTHS[g] + 1) for g in game])
    err = check(net, game, length)
    check(net, game, length, grad=False)
    print(f"H={net[1][1]} layers={net[1][2]}: max relative gradient error {err:.2e}")


def test_labels_of_rows_that_are_no_permutation(net):
    rank = np.array([[0, 0, 1, 2], [3, 2, 1, 0], [4, 1, 2, 3], [1, 0, 3, 2]])
    check(net, [0, 1, 2, 3], [1, 2, 5, 20], rank=rank)


def test_argument_checks():
    grp = T.random_grp(8, 2, 1)
    w, h, nl = T.pack(grp)
    rng = np.random.default_rng(0)
    f = [T.random_feature(3, rng), T.random_feature(5, rng)]
    game, length, rank = [0, 1, 1], [3, 2, 5], [[0, 1, 2, 3]] * 3
    assert T.run_emul(w, h, nl, f, game, length, rank)[0] == 0
    assert T.run_emul(w, h, nl, f, game, length, rank, n_weights=w.size - 1)[0] == -2
    for hid, lay in ((0, 1), (257, 1), (8, 0), (8, 5)):
        assert T.run_emul(w, hid, lay, f, game, length, rank)[0] == -2, (hid, lay)
    assert T.run_emul(w, h, nl, f, game, length, rank, n_rows=0)[0] == -2
    assert T.run_emul(w, h, nl, f, game, length, rank, n_samples=0)[0] == -2
    assert T.run_emul(w, h, nl, f, game, length, rank, scratch_bytes=8)[0] == -2
    L = T.emul_lib()
    assert L.emult_scratch_bytes(8, 2, 3, 4, 5) == -2  # more jobs than samples
    assert L.emult_scratch_bytes(8, 2, 3, 2, 0) == -2
    assert T.run_emul(*T.pack(T.random_grp(256, 4, 2)), f, game, length, rank)[0] == 0  # the largest shape


def test_sample_statuses():
    grp = T.random_grp(8, 2, 4)
    w, h, nl = T.pack(grp)
    rng = np.random.default_rng(2)
    f = [T.random_feature(n, rng) for n in (3, 5, 4)]
    game = np.array([0, 1, 1, 2, 2, 0])
    length = np.array([3, 2, 5, 4, 1, 2])
    rank = np.array([rng.permutation(4) for _ in game])
    jobs = T.jobs_of(game, length)
    bad_game = game.copy()
    bad_game[1] = 7                   # not its job's game
    bad_len = length.copy()
    bad_len[4] = 0                    # length 0
    jobs["job_steps"] = jobs["job_steps"].copy()
    rc, loss, acc, g, status = T.run_emul(w, h, nl, f, bad_game, bad_len, rank, jobs=jobs)
    assert rc == 0 and status.tolist() == [0, 1, 0, 0, 2, 0]
    # the bad samples contribute nothing: the loss is the sum over the good ones / B
    keep = [0, 2, 3, 5]
    inputs = [torch.as_tensor(f[a][:b]) for a, b in zip(game[keep], length[keep])]
    want_loss, _ = T.ref_step(grp, inputs, rank[keep])
    assert abs(loss - want_loss * 4 / 6) <= 1e-12 * abs(want_loss)
    assert T.grad_err(g * 6 / 4, grp) <= 1e-12
    # a job whose steps exceed its game: its samples get GAME; a game whose offsets lie outside the rows likewise
    jobs2 = T.jobs_of(game, length)
    jobs2["job_steps"][0] = 9
    status = T.run_emul(w, h, nl, f, game, length, rank, jobs=jobs2)[4]
    assert status.tolist() == [1, 0, 0, 0, 0, 1]
    packed = dict(feat=np.concatenate(f), game_off=np.array([0, 3, 8, 20], dtype=np.int32))
    status = T.run_emul(w, h, nl, packed, game, length, rank)[4]
    assert status.tolist() == [0, 0, 0, 1, 1, 0]
