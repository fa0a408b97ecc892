"""GameplayLoader on single-viewpoint logs (k_replay_viewpoints, mjx_env_replay_viewpoints): the copy of an arena log that the mjai
protocol shows one seat (the other seats' haipai and draws are "?") loads for that seat to exactly the Gameplays of the full log,
through the device decoder and through the host path; full logs in the same batch are untouched; a log whose own seat is hidden
fails with code 13 on both paths; oracle=True still refuses such logs; Grp and Stat read them as they read the full logs."""
import gzip
import json
import os

import numpy as np
import pytest

from viewpoint_lib import named, viewpoint

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


class _Eng:
    engine_type, version, is_oracle, enable_quick_eval, enable_rule_based_agari_guard = "mortal", 4, False, True, False

    def __init__(self, name, bias):
        self.name, self.bias = name, bias

    def react_device(self, obs, masks):
        q = torch.rand(masks.shape, device=masks.device)
        q[:, :34] += self.bias * obs[:, 876, :] + obs[:, 875, :]
        q = q.masked_fill(~masks, -1.0)
        return q.argmax(-1), q


def _write(path, events):
    with gzip.open(path, "wt") as f:
        f.write("".join(json.dumps(ev) + "\n" for ev in events))


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    """256 arena logs of two engines: full/ holds each log with distinct seat names, view<p>/ the same logs as seat p sees them"""
    from mortal_b200.libriichi.arena import OneVsThree

    arena = tmp_path_factory.mktemp("vp_arena")
    torch.manual_seed(5)
    OneVsThree(disable_progress_bar=True, log_dir=str(arena)).py_vs_py(_Eng("alpha", 2.0), _Eng("beta", 0.5), (93000, 31), 64)
    src = sorted(os.path.join(arena, f) for f in os.listdir(arena))
    assert len(src) == 256
    root = tmp_path_factory.mktemp("vp_logs")
    out = {"full": []} | {p: [] for p in range(4)}
    for d in ["full"] + [f"view{p}" for p in range(4)]:
        os.makedirs(root / d)
    for k, fn in enumerate(src):
        with gzip.open(fn, "rt") as f:
            ev = [json.loads(ln) for ln in f if ln.strip()]
        out["full"].append(str(root / "full" / f"{k:04d}.json.gz"))
        _write(out["full"][-1], named(ev))
        for p in range(4):
            out[p].append(str(root / f"view{p}" / f"{k:04d}.json.gz"))
            _write(out[p][-1], viewpoint(ev, p))
    out["root"] = root
    return out


def _seat(p):
    """player_names selecting seat p of named() logs, whichever engine sat there"""
    return [f"alpha.{p}", f"beta.{p}"]


def _host(monkeypatch, fn):
    from mortal_b200 import _logio

    with monkeypatch.context() as m:
        m.setattr(_logio, "device_ready", lambda: False)
        return fn()


def _outcome(fn):
    try:
        return fn()
    except Exception as e:  # noqa: BLE001
        return (type(e), str(e))


def _same_grp(a, b):
    fa, fb = a.take_feature(), b.take_feature()
    assert fa.dtype == fb.dtype == np.float64 and fa.shape == fb.shape and np.array_equal(fa, fb)
    assert a.take_rank_by_player() == b.take_rank_by_player() and a.take_final_scores() == b.take_final_scores()


def _same(got, want):
    """every Gameplay field, bit for bit"""
    assert len(got) == len(want)
    n = 0
    for pg, pw in zip(got, want):
        assert len(pg) == len(pw)
        for a, b in zip(pg, pw):
            assert a.take_player_id() == b.take_player_id() and a.player_name == b.player_name
            oa, ob = a.take_obs(), b.take_obs()
            assert oa.shape == ob.shape and torch.equal(oa.cpu(), ob.cpu()) and torch.equal(a.take_masks().cpu(), b.take_masks().cpu())
            for f in ("take_actions", "take_at_kyoku", "take_dones", "take_apply_gamma", "take_at_turns", "take_shantens"):
                assert getattr(a, f)() == getattr(b, f)(), f
            _same_grp(a.take_grp(), b.take_grp())
            n += len(a.take_actions())
    return n


def test_viewpoint_logs_load_to_the_full_logs_gameplays(corpus):
    from mortal_b200.dataset import GameplayLoader

    moves = 0
    for p in range(4):
        for lo in range(0, 256, 64):  # 64 logs per call: bounded device memory for the observations
            kw = dict(oracle=False, player_names=_seat(p))
            got = GameplayLoader(4, **kw).load_gz_log_files(corpus[p][lo:lo + 64])
            want = GameplayLoader(4, **kw).load_gz_log_files(corpus["full"][lo:lo + 64])
            assert all(len(g) == 1 and g[0].take_player_id() == p for g in got)
            moves += _same(got, want)
    assert moves > 50000


@pytest.mark.parametrize("kw", [dict(), dict(augmented=True), dict(always_include_kan_select=False)], ids=["plain", "augmented", "no kan select"])
@pytest.mark.parametrize("version", [1, 2, 3])
def test_viewpoint_logs_other_settings(corpus, version, kw):
    from mortal_b200.dataset import GameplayLoader

    for p in (0, 3):
        a = GameplayLoader(version, oracle=False, player_names=_seat(p), **kw)
        _same(a.load_gz_log_files(corpus[p][:12]), a.load_gz_log_files(corpus["full"][:12]))


def test_both_paths_and_a_real_device_decode(corpus, monkeypatch):
    """the host path (forced) gives the device path's result on the masked files, and the device path takes none of them to the
    host parser"""
    from mortal_b200 import dataset_codec
    from mortal_b200.dataset import GameplayLoader

    files = {p: corpus[p][100:124] for p in range(4)}
    want = {p: _host(monkeypatch, lambda: GameplayLoader(4, oracle=False, player_names=_seat(p)).load_gz_log_files(files[p]))
            for p in range(4)}

    def no_parse(text):
        raise AssertionError("a log went to the host parser")

    with monkeypatch.context() as m:
        m.setattr(dataset_codec, "parse_log", no_parse)
        for p in range(4):
            _same(GameplayLoader(4, oracle=False, player_names=_seat(p)).load_gz_log_files(files[p]), want[p])
            _same(GameplayLoader(4, oracle=False, player_names=_seat(p)).load_gz_log_files(files[p]),
                  GameplayLoader(4, oracle=False, player_names=_seat(p)).load_gz_log_files(corpus["full"][100:124]))


def test_mixed_batches(corpus, monkeypatch):
    from mortal_b200.dataset import GameplayLoader

    full, masked = corpus["full"][130:138], corpus[2][138:146]
    # full and masked logs together: the full logs' rows are those of loading them alone
    kw = dict(oracle=False, player_names=_seat(2))
    both = GameplayLoader(4, **kw).load_gz_log_files(full[:4] + masked + full[4:])
    _same(both[:4] + both[-4:], GameplayLoader(4, **kw).load_gz_log_files(full))
    _same(both[4:-4], GameplayLoader(4, **kw).load_gz_log_files(corpus["full"][138:146]))
    # the default player selection (all four seats) on a masked log: code 13, the same job number on both paths
    files = full[:2] + [corpus[1][140]] + full[2:3]
    got = _outcome(lambda: GameplayLoader(4, oracle=False).load_gz_log_files(files))
    want = _outcome(lambda: _host(monkeypatch, lambda: GameplayLoader(4, oracle=False).load_gz_log_files(files)))
    assert got == want and got[0] is RuntimeError, (got, want)
    assert "replay job 8 (log 2, player 0)" in got[1] and "code 13" in got[1] and "own tiles are hidden" in got[1], got
    assert "player_names" in got[1]


def test_oracle_loads_still_refuse_masked_logs(corpus):
    from mortal_b200.dataset import GameplayLoader

    for trust_seed in (True, False):
        with pytest.raises(Exception):
            GameplayLoader(4, oracle=True, trust_seed=trust_seed, player_names=_seat(1)).load_gz_log_files(corpus[1][:2])
    # and the full logs still load with oracle=True
    assert len(GameplayLoader(4, oracle=True, trust_seed=True, player_names=_seat(1)).load_gz_log_files(corpus["full"][:2])) == 2


def test_grp_and_stat_read_masked_logs_as_full_logs(corpus):
    from mortal_b200.dataset import Grp
    from mortal_b200.stat import COUNTERS, Stat

    want = Grp.load_gz_log_files(corpus["full"])
    for p in range(4):
        for a, b in zip(Grp.load_gz_log_files(corpus[p]), want):
            _same_grp(a, b)
    root = corpus["root"]
    for p in range(4):
        for nm in (f"alpha.{p}", f"beta.{p}"):
            a, b = Stat.from_dir(str(root / f"view{p}"), nm), Stat.from_dir(str(root / "full"), nm)
            assert all(getattr(a, c) == getattr(b, c) for c in COUNTERS) and a.game > 0, (p, nm)


def test_replay_env_viewpoints_call_order(corpus):
    """mjx_env_replay_viewpoints: not with trust_seeds (either order) and only before the first step"""
    from mortal_b200 import _lib, dataset_codec
    from mortal_b200.env import ReplayEnv

    with gzip.open(corpus[0][0], "rt") as f:
        ev = dataset_codec.parse_log(f.read())
    jobs = dataset_codec.build_jobs([ev], [[0]])
    env = ReplayEnv(jobs)
    env.trust_seeds([1], [2])
    with pytest.raises(_lib.MjxError, match="trust_seeds"):
        env.viewpoints()
    env.close()
    env = ReplayEnv(jobs)
    env.viewpoints()
    with pytest.raises(_lib.MjxError, match="viewpoints"):
        env.trust_seeds([1], [2])
    env.replay_step()
    with pytest.raises(_lib.MjxError, match="before the first"):
        env.viewpoints()
    env.close()
