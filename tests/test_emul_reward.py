"""k_grp_matrix and k_train_targets (csrc/mjx_reward.cuh, host build) against a torch-CPU float64 restatement of the reference:
the rank-probability matrix of every prefix equals the O(L^2) prefix-list formulation of reward_calculator.py within 1e-12, the
kyoku rewards within 1e-10, and steps_to_done / player ranks of dataloader.py populate_buffer exactly; bad arguments and bad job
arrays give the documented codes."""
import numpy as np
import pytest
import torch

import reward_lib as R

LENGTHS = (1, 2, 8, 20, 40, 64)
PTS = ((3, 1, -1, -3), (90, 45, 0, -135))


@pytest.fixture(scope="module", params=[(64, 2), (32, 1), (96, 3)], ids=lambda p: f"H{p[0]}xL{p[1]}")
def net(request):
    hidden, layers = request.param
    grp = R.random_grp(hidden, layers, 100 + hidden + layers)
    rng = np.random.default_rng(hidden * 10 + layers)
    feats = [R.random_feature(n, rng) for n in LENGTHS]
    return grp, R.pack(grp), feats, [R.ref_calc_grp(grp, f) for f in feats]


def test_matrix_matches_prefix_list_reference(net):
    grp, (w, h, nl), feats, want = net
    rc, m, *_ = R.run_emul(w, h, nl, feats)
    assert rc == 0
    off = np.cumsum([0] + [len(f) for f in feats])
    err = max(np.abs(m[off[i]:off[i + 1]] - want[i].numpy()).max() for i in range(len(feats)))
    probs = np.concatenate([x.numpy().reshape(-1) for x in want])
    print(f"H={h} layers={nl}: max |matrix - reference| = {err:.3e} (entries {probs.min():.3f}..{probs.max():.3f})")
    assert err <= 1e-12
    assert probs.min() < 0.1 and probs.max() > 0.45  # the softmax is neither flat nor one-hot


@pytest.mark.parametrize("uniform_init", [False, True])
@pytest.mark.parametrize("pts", PTS)
def test_rewards_and_targets(net, pts, uniform_init):
    grp, (w, h, nl), feats, mats = net
    rng = np.random.default_rng(7)
    ranks = [rng.permutation(4) for _ in feats]
    finals = [(f[-1, 3:] * 1e4).astype(np.int64) + rng.integers(-20, 20, size=4) * 100 for f in feats]
    for g in range(0, len(finals), 3):
        finals[g][2] = finals[g][0]  # a tie in the final row
    # calc_delta_pt's jobs (one per game and player, its moves the kyoku) and Gameplay-like jobs of random moves
    gps = [(p, np.arange(len(f)), np.ones(len(f), dtype=bool), np.zeros(len(f), dtype=bool), g) for g, f in enumerate(feats)
           for p in range(4)]
    gps += [R.random_gameplay(len(f), rng, int(rng.integers(0, 4)), g) for g, f in enumerate(feats) for _ in range(2)]
    jobs = R.jobs_of(gps, feats, ranks, finals)
    rc, _, steps, reward, rank, status = R.run_emul(w, h, nl, feats, jobs, pts=pts, uniform_init=uniform_init)
    assert rc == 0 and not status.any()
    err = 0.0
    for j, (pid, at_kyoku, dones, apply_gamma, g) in enumerate(gps):
        sl = slice(jobs["move_off"][j], jobs["move_off"][j + 1])
        kr = R.ref_delta_pt(mats[g], list(pts), uniform_init, pid, ranks[g])
        ws, wr, wk = R.ref_targets(kr, pid, feats[g], finals[g], at_kyoku, dones, apply_gamma)
        assert np.array_equal(steps[sl], ws) and np.array_equal(rank[sl], wk), j
        err = max(err, np.abs(reward[sl] - wr).max())
    print(f"H={h} layers={nl} pts={pts} uniform_init={uniform_init}: max |reward - reference| = {err:.3e}")
    assert err <= 1e-10


def test_argument_checks():
    grp = R.random_grp(8, 1, 1)
    w, h, nl = R.pack(grp)
    f = [R.random_feature(3, np.random.default_rng(0))]
    assert R.run_emul(w, h, nl, f)[0] == 0
    assert R.run_emul(w, h, nl, f, n_weights=w.size - 1)[0] == -2
    for hid, lay in ((0, 1), (257, 1), (8, 0), (8, 5)):
        assert R.run_emul(w, hid, lay, f)[0] == -2, (hid, lay)
    assert R.run_emul(w, h, nl, [])[0] == -2  # no games
    big = R.pack(R.random_grp(256, 4, 2))
    assert R.run_emul(*big, f)[0] == 0  # the largest shape


def test_job_statuses():
    grp = R.random_grp(16, 2, 3)
    w, h, nl = R.pack(grp)
    rng = np.random.default_rng(5)
    feats = [R.random_feature(n, rng) for n in (4, 6)]
    gps = [R.random_gameplay(len(feats[g]), rng, p, g) for g, p in ((0, 0), (1, 3), (0, 2), (1, 1), (0, 1))]
    jobs = R.jobs_of(gps, feats, [[0, 1, 2, 3], [3, 2, 1, 0]], [[25000] * 4, [30000, 20000, 25000, 25000]])
    jobs["at_kyoku"][jobs["move_off"][1]] = 6  # job 1: a kyoku past its game's 6 rows
    jobs["job_game"][2] = 2                    # job 2: no such game
    jobs["job_player"][3] = 4                  # job 3: no such seat
    rc, _, steps, reward, rank, status = R.run_emul(w, h, nl, feats, jobs)
    assert rc == 0 and status.tolist() == [0, 2, 1, 1, 0]
    sl = slice(jobs["move_off"][1], jobs["move_off"][2])
    assert not steps[sl].any() and not reward[sl].any() and not rank[sl].any()
    sl = slice(jobs["move_off"][2], jobs["move_off"][4])
    assert (steps[sl] == -7).all() and (rank[sl] == -7).all()  # CAPACITY writes nothing
    # a game whose offsets lie outside the rows: no matrix rows, its jobs CAPACITY
    packed = dict(feat=np.concatenate(feats), game_off=np.array([0, 4, 11], dtype=np.int32))
    rc, m, *_, status = R.run_emul(w, h, nl, packed, jobs)
    assert rc == 0 and np.isnan(m[4:]).all() and not np.isnan(m[:4]).any()
    assert status[1] == 1 and status[3] == 1 and status[0] == 0


def test_weight_layout_rejects_bad_state_dicts():
    from mortal_b200.reward import pack_grp_weights

    for hid, lay in ((257, 1), (8, 5)):
        with pytest.raises(ValueError):
            pack_grp_weights(R.RefGRP(hid, lay).state_dict())
    sd = R.RefGRP(8, 2).state_dict()
    sd["fc.2.weight"] = torch.zeros(23, 16, dtype=torch.float64)
    with pytest.raises(ValueError):
        pack_grp_weights(sd)
