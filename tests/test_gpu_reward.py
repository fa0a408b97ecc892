"""mortal_b200.reward on the device (k_grp_matrix, k_train_targets): RewardCalculator against a torch-CPU float64 restatement of
reward_calculator.py (the O(L^2) prefix-list formulation), training_samples against a restatement of dataloader.py populate_buffer
on arena logs loaded by GameplayLoader (oracle=False and oracle=True, trust_seed=True), calc_delta_pt_batch over the arena's
recorded GRP features, and the edge cases: one-kyoku and 64-kyoku games, Gameplays without moves, the reference's assertion,
unsupported net shapes."""
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import reward_lib as R  # noqa: E402
from test_gpu_gameplay_decode import _Eng  # noqa: E402

LENGTHS = (1, 2, 8, 20, 40, 64)


@pytest.fixture(scope="module")
def grp():
    return R.random_grp(64, 2, 11)


@pytest.mark.parametrize("shape", [(64, 2), (32, 1), (96, 3)], ids=lambda p: f"H{p[0]}xL{p[1]}")
def test_calc_methods_match_reference(shape):
    from mortal_b200.reward import RewardCalculator

    net = R.random_grp(*shape, 200 + shape[0])
    rng = np.random.default_rng(shape[0])
    feats = [R.random_feature(n, rng) for n in LENGTHS]
    mats = [R.ref_calc_grp(net, f) for f in feats]
    err_m = err_r = 0.0
    for pts, uniform_init in (((3, 1, -1, -3), False), ([90, 45, 0, -135], False), ([90, 45, 0, -135], True), (None, True)):
        rc = RewardCalculator(net if uniform_init else net.state_dict(), list(pts) if pts else None, uniform_init)
        for f, m in zip(feats, mats):
            got = rc.calc_grp(f)
            assert got.is_cuda and got.dtype == torch.float64 and got.shape == (len(f), 4, 4)
            err_m = max(err_m, (got.cpu() - m).abs().max().item())
            rank = [int(x) for x in rng.permutation(4)]
            for pid in range(4):
                rp = rc.calc_rank_prob(pid, f, rank)
                want_rp = R.ref_rank_prob(m, uniform_init, pid, rank)
                assert rp.shape == want_rp.shape and (rp.cpu() - want_rp).abs().max().item() <= 1e-12
                d = rc.calc_delta_pt(pid, f, rank)
                want = R.ref_delta_pt(m, list(pts) if pts else None, uniform_init, pid, rank)
                assert isinstance(d, np.ndarray) and d.dtype == np.float64 and d.shape == (len(f),)
                err_r = max(err_r, np.abs(d - want).max())
            fs = [25000, 25000, 25000, 25000]
            assert np.array_equal(rc.calc_delta_points(1, f, fs), np.diff(np.append(f[:, 4] * 1e4, fs[1])))
    print(f"H={shape[0]} layers={shape[1]}: max |matrix - reference| = {err_m:.3e}, max |reward - reference| = {err_r:.3e}")
    assert err_m <= 1e-12 and err_r <= 1e-10


def ref_samples(data, net, pts, oracle):
    """dataloader.py populate_buffer restated over a GameplayLoader result with the CPU reference GRP (one calc_grp per Gameplay,
    as the reference runs it) -> the buffer's columns"""
    cols = {k: [] for k in ("obs", "invisible_obs", "actions", "masks", "steps_to_done", "kyoku_rewards", "player_ranks")}
    for file in data:
        for game in file:
            at_kyoku = game.take_at_kyoku()
            if not at_kyoku:
                continue
            grp = game.take_grp()
            pid = game.take_player_id()
            kr = R.ref_delta_pt(R.ref_calc_grp(net, grp.take_feature()), pts, False, pid, grp.take_rank_by_player())
            s, r, k = R.ref_targets(kr, pid, grp.take_feature(), grp.take_final_scores(), at_kyoku, game.take_dones(),
                                    game.take_apply_gamma())
            cols["obs"].append(game.take_obs()); cols["masks"].append(game.take_masks())
            if oracle:
                cols["invisible_obs"].append(game.take_invisible_obs())
            cols["actions"].append(np.array(game.take_actions(), dtype=np.int64))
            cols["steps_to_done"].append(s); cols["kyoku_rewards"].append(r); cols["player_ranks"].append(k)
    return cols


@pytest.fixture(scope="module")
def arena_files(tmp_path_factory):
    from mortal_b200.libriichi.arena import OneVsThree

    d = tmp_path_factory.mktemp("arena_reward")
    torch.manual_seed(5)
    OneVsThree(disable_progress_bar=True, log_dir=str(d)).py_vs_py(_Eng("alpha", 2.0), _Eng("beta", 0.5), (93000, 31), 64)
    files = sorted(os.path.join(d, f) for f in os.listdir(d))
    assert len(files) == 256
    return files


@pytest.mark.parametrize("oracle", [False, True], ids=["visible", "oracle"])
def test_training_samples_match_populate_buffer(arena_files, grp, oracle):
    from mortal_b200.dataset import GameplayLoader
    from mortal_b200.reward import RewardCalculator, training_samples

    loader = GameplayLoader(4, oracle=oracle, trust_seed=oracle)
    rc = RewardCalculator(grp, [90, 45, 0, -135])
    err, n = 0.0, 0
    for b in range(0, len(arena_files), 32):
        data = loader.load_gz_log_files(arena_files[b:b + 32])
        got = training_samples(data, rc)
        want = ref_samples(data, grp, [90, 45, 0, -135], oracle)
        assert set(got) == {"obs", "actions", "masks", "steps_to_done", "kyoku_rewards", "player_ranks"} | ({"invisible_obs"} if oracle else set())
        for k in ("obs", "masks") + (("invisible_obs",) if oracle else ()):
            assert got[k].is_cuda and torch.equal(got[k], torch.cat(want[k])), k
        for k in ("actions", "steps_to_done", "player_ranks"):
            assert got[k].dtype == torch.int64 and np.array_equal(got[k].cpu().numpy(), np.concatenate(want[k])), k
        assert got["kyoku_rewards"].dtype == torch.float64
        err = max(err, np.abs(got["kyoku_rewards"].cpu().numpy() - np.concatenate(want["kyoku_rewards"])).max())
        n += len(got["actions"])
        del data, got, want
    print(f"oracle={oracle}: {n} samples from {len(arena_files)} files, max |kyoku reward - reference| = {err:.3e}")
    assert err <= 1e-10


def test_calc_delta_pt_batch_over_arena_grp(grp):
    from mortal_b200.libriichi.arena import OneVsThree
    from mortal_b200.reward import RewardCalculator

    arena = OneVsThree(disable_progress_bar=True)
    arena.record_grp = True
    torch.manual_seed(6)
    arena.py_vs_py(_Eng("alpha", 2.0), _Eng("beta", 0.5), (94000, 37), 16)
    grps = arena.last_grp
    assert len(grps) == 64
    rng = np.random.default_rng(3)
    pids = rng.integers(0, 4, size=len(grps))
    rc = RewardCalculator(grp, None, True)
    rewards, offsets = rc.calc_delta_pt_batch(pids.tolist(), grps)
    assert rewards.is_cuda and rewards.dtype == torch.float64 and offsets.dtype == torch.int64 and len(offsets) == len(grps) + 1
    got = rewards.cpu().numpy()
    for i, g in enumerate(grps):
        want = R.ref_delta_pt(R.ref_calc_grp(grp, g.take_feature()), None, True, int(pids[i]), g.take_rank_by_player())
        assert np.abs(got[offsets[i]:offsets[i + 1]] - want).max() <= 1e-10, i


def _gameplay(grp_obj, pid, at_kyoku, dev, seed):
    from mortal_b200.dataset import Gameplay

    g = torch.Generator(device="cpu").manual_seed(seed)
    n = len(at_kyoku)
    at_kyoku = np.asarray(at_kyoku, dtype=np.uint8)
    return Gameplay(pid, "p", torch.rand((n, 5, 34), generator=g).to(dev), np.arange(n, dtype=np.int64) % 46,
                    (torch.rand((n, 46), generator=g) < 0.5).to(dev), at_kyoku, np.arange(n) % 3 != 0, np.zeros(n, dtype=np.uint8),
                    np.zeros(n, dtype=np.int8), grp=grp_obj)


def test_edge_cases(grp):
    from mortal_b200.dataset import Grp
    from mortal_b200.reward import RewardCalculator, training_samples

    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(9)
    rc = RewardCalculator(grp)
    one = Grp(R.random_feature(1, rng), [2, 0, 3, 1], [24000, 41000, 10000, 25000])
    long = Grp(R.random_feature(64, rng), [0, 1, 2, 3], [40000, 30000, 20000, 10000])  # more kyoku than the arena records
    at_long = np.repeat(np.arange(64), rng.integers(0, 4, size=64))
    at_long[-1] = 63
    data = [[_gameplay(one, 0, [0, 0, 0], dev, 1), _gameplay(one, 2, [], dev, 2), _gameplay(one, 3, [0], dev, 3)],
            [_gameplay(long, 1, at_long, dev, 4)], [_gameplay(long, 2, [], dev, 5)]]
    got = training_samples(data, rc)
    want = ref_samples(data, grp, None, False)
    assert len(got["actions"]) == 4 + len(at_long)  # the Gameplays without moves give no samples
    for k in ("steps_to_done", "player_ranks", "actions"):
        assert np.array_equal(got[k].cpu().numpy(), np.concatenate(want[k])), k
    assert np.abs(got["kyoku_rewards"].cpu().numpy() - np.concatenate(want["kyoku_rewards"])).max() <= 1e-10
    assert torch.equal(got["obs"], torch.cat(want["obs"])) and torch.equal(got["masks"], torch.cat(want["masks"]))
    # nothing but Gameplays without moves
    empty = training_samples([[_gameplay(one, 0, [], dev, 6)]], rc)
    assert all(v.shape[0] == 0 for v in empty.values())
    # the reference's assertion: a move in a kyoku the game's rows do not reach
    with pytest.raises(AssertionError):
        training_samples([[_gameplay(one, 0, [0, 1], dev, 7)]], rc)
    # unsupported shapes
    for shape in ((300, 1), (16, 5)):
        with pytest.raises(ValueError):
            RewardCalculator(R.RefGRP(*shape))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_device_other_than_current(grp):
    from mortal_b200.reward import RewardCalculator

    f = R.random_feature(12, np.random.default_rng(4))
    want = R.ref_delta_pt(R.ref_calc_grp(grp, f), None, False, 1, [1, 0, 2, 3])
    with torch.cuda.device(0):
        rc = RewardCalculator(grp, device=1)
        m = rc.calc_grp(f)
        assert m.device == torch.device("cuda", 1)
        assert np.abs(rc.calc_delta_pt(1, f, [1, 0, 2, 3]) - want).max() <= 1e-10
