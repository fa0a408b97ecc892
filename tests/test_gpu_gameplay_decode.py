"""GameplayLoader and Grp.load_gz_log_files on the device decoder (k_mjai_decode with the deltas output, k_grp_logs, the replay
from device arrays): every Gameplay field and every Grp equals what the host path, forced in the same process, returns; the
device really decodes; batches with logs the decoder declines at the start, middle and end give the same result; bad batches raise
the host path's exception with its message; Grp.load_gz_log_files runs on libmjx's device."""
import gzip
import json
import os

import numpy as np
import pytest

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


@pytest.fixture(scope="module")
def arena_files(tmp_path_factory):
    from mortal_b200.libriichi.arena import OneVsThree

    d = tmp_path_factory.mktemp("arena_loader")
    torch.manual_seed(3)
    OneVsThree(disable_progress_bar=True, log_dir=str(d)).py_vs_py(_Eng("alpha", 2.0), _Eng("beta", 0.5), (91000, 29), 256)
    files = sorted(os.path.join(d, f) for f in os.listdir(d))
    assert len(files) == 1024
    return files


@pytest.fixture(scope="module")
def arena_texts(arena_files):
    return [gzip.open(f, "rt").read() for f in arena_files[:24]]


def _host(monkeypatch, fn):
    """fn() with the device path switched off: today's host code end to end"""
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
    assert all(type(x) is int for x in a.take_rank_by_player() + a.take_final_scores())


def _same(got, want, oracle=False):
    assert len(got) == len(want)
    for pg, pw in zip(got, want):
        assert len(pg) == len(pw)
        for a, b in zip(pg, pw):
            assert a.take_player_id() == b.take_player_id() and a.player_name == b.player_name
            assert torch.equal(a.take_obs().cpu(), b.take_obs().cpu()) and torch.equal(a.take_masks().cpu(), b.take_masks().cpu())
            if oracle:
                assert torch.equal(a.take_invisible_obs().cpu(), b.take_invisible_obs().cpu())
            for f in ("take_actions", "take_at_kyoku", "take_dones", "take_apply_gamma", "take_at_turns", "take_shantens"):
                assert getattr(a, f)() == getattr(b, f)(), f
            _same_grp(a.take_grp(), b.take_grp())
        if pg:
            assert all(gp.take_grp() is pg[0].take_grp() for gp in pg)  # one Grp per log, shared by its players


def test_device_path_is_taken():
    from mortal_b200 import _logio
    from mortal_b200.dataset import GameplayLoader

    assert _logio.device_ready()
    assert GameplayLoader(4, oracle=False)._on_device() and GameplayLoader(4, trust_seed=True)._on_device()
    assert not GameplayLoader(4, oracle=True, trust_seed=False)._on_device()


SETTINGS = {
    "v4": dict(oracle=False),
    "augmented": dict(oracle=False, augmented=True),
    "player_names": dict(oracle=False, player_names=["alpha"]),
    "excludes": dict(oracle=False, excludes=["alpha"]),
    "nobody selected": dict(oracle=False, player_names=["nobody"]),
    "oracle, trust_seed": dict(oracle=True, trust_seed=True),
}


@pytest.mark.parametrize("name", list(SETTINGS))
def test_loader_equals_the_host_path(arena_files, monkeypatch, name):
    from mortal_b200.dataset import GameplayLoader

    kw = SETTINGS[name]
    files = arena_files[:20]
    got = GameplayLoader(4, **kw).load_gz_log_files(files)
    want = _host(monkeypatch, lambda: GameplayLoader(4, **kw).load_gz_log_files(files))
    _same(got, want, oracle=kw["oracle"])
    assert sum(len(g) for g in got) == {"player_names": 20, "excludes": 60, "nobody selected": 0}.get(name, 80)


def test_the_device_really_decodes(arena_files, monkeypatch):
    """with the host parser disabled, arena logs still load (plain and augmented) and their Grp still comes back"""
    from mortal_b200 import dataset_codec
    from mortal_b200.dataset import GameplayLoader, Grp

    files = arena_files[20:28]
    want = {aug: _host(monkeypatch, lambda: GameplayLoader(4, oracle=False, augmented=aug).load_gz_log_files(files))
            for aug in (False, True)}
    want_grp = _host(monkeypatch, lambda: Grp.load_gz_log_files(files))

    def no_parse(text):
        raise AssertionError("a log went to the host parser")

    monkeypatch.setattr(dataset_codec, "parse_log", no_parse)
    for aug in (False, True):
        _same(GameplayLoader(4, oracle=False, augmented=aug).load_gz_log_files(files), want[aug])
    for a, b in zip(Grp.load_gz_log_files(files), want_grp):
        _same_grp(a, b)


def _declined(text, kind):
    """an arena log rewritten so that the decoder declines it while Python reads the same events"""
    lines = text.splitlines()
    if kind == "lone CR":
        return "\r".join(lines[:3]) + "\n" + "\n".join(lines[3:]) + "\n"
    first = json.loads(lines[0])
    if kind == "NaN":
        lines[0] = lines[0][:-1] + ', "x": NaN}'
    elif kind == "duplicated key":
        lines[-1] = '{"type":"end_game","type":"end_game"}'
    elif kind == "not UTF-8":
        lines[0] = lines[0][:-1] + ', "x": "\udcff"}'
    assert json.loads(lines[0])["type"] == first["type"]
    return "\n".join(lines) + "\n"


@pytest.mark.parametrize("augmented", [False, True])
def test_mixed_batches_equal_the_host_path(arena_texts, monkeypatch, augmented):
    from mortal_b200.dataset import GameplayLoader

    t = arena_texts
    texts = ([_declined(t[0], "lone CR"), t[1], t[2], _declined(t[3], "NaN"), t[4], _declined(t[5], "duplicated key"), t[6],
              _declined(t[7], "not UTF-8")])
    kw = dict(oracle=False, augmented=augmented)
    got = GameplayLoader(4, **kw).load_logs(texts)
    _same(got, _host(monkeypatch, lambda: GameplayLoader(4, **kw).load_logs(texts)))
    for text in (texts[1], texts[3]):
        _same([GameplayLoader(4, **kw).load_log(text)], [_host(monkeypatch, lambda: GameplayLoader(4, **kw).load_log(text))])


def test_mixed_files_equal_the_host_path(arena_texts, tmp_path, monkeypatch):
    """declined files among accepted ones, including a lone CR the text reader turns into a newline"""
    from mortal_b200.dataset import GameplayLoader, Grp

    texts = [_declined(arena_texts[8], "lone CR"), arena_texts[9], _declined(arena_texts[10], "NaN"), arena_texts[11]]
    files = []
    for k, text in enumerate(texts):
        files.append(str(tmp_path / f"{k}.json.gz"))
        with gzip.open(files[-1], "wb") as f:
            f.write(text.encode("utf-8"))
    _same(GameplayLoader(4, oracle=False).load_gz_log_files(files),
          _host(monkeypatch, lambda: GameplayLoader(4, oracle=False).load_gz_log_files(files)))
    for a, b in zip(Grp.load_gz_log_files(files), _host(monkeypatch, lambda: Grp.load_gz_log_files(files))):
        _same_grp(a, b)


def _without_final_deltas(text):
    lines = text.splitlines()
    k = max(i for i, ln in enumerate(lines) if json.loads(ln)["type"] in ("hora", "ryukyoku"))
    ev = json.loads(lines[k])
    del ev["deltas"]
    lines[k] = json.dumps(ev)
    return "\n".join(lines) + "\n"


def _with_seed(text, seed):
    lines = text.splitlines()
    ev = json.loads(lines[0])
    ev["seed"] = seed
    lines[0] = json.dumps(ev)
    return "\n".join(lines) + "\n"


def test_bad_batches_raise_the_host_exception(arena_texts, monkeypatch):
    from mortal_b200.dataset import GameplayLoader

    t = arena_texts[12:16]
    lines = t[0].splitlines()
    bad = {
        "first line not JSON": [t[1], lines[0][:-1] + "\n" + "\n".join(lines[1:]), t[2]],
        "first event not start_game": [t[1], "\n".join(lines[1:]), t[2]],
        "fewer than 4 events": [t[1], "\n".join(lines[:2] + lines[-1:]), t[2]],
        "only blank lines": [t[1], " \n\t\n", t[2]],
        "a parse error after a short log": ["\n".join(lines[:3]), t[1], "{"],
        "missing final deltas": [t[1], _without_final_deltas(t[2]), t[3]],
        "missing final deltas, declined by the decoder": [t[1], _declined(_without_final_deltas(t[2]), "NaN"), t[3]],
    }
    for name, texts in bad.items():
        for kw in (dict(oracle=False), dict(oracle=False, augmented=True)):
            got = _outcome(lambda: GameplayLoader(4, **kw).load_logs(texts))
            want = _outcome(lambda: _host(monkeypatch, lambda: GameplayLoader(4, **kw).load_logs(texts)))
            assert isinstance(want, tuple) and got == want, (name, kw, got, want)
    # a replay error: the third log's seed does not deal its hands; the job number counts logs, then players
    seeded = [t[0], t[1], _with_seed(t[2], [1, 2]), t[3]]
    got = _outcome(lambda: GameplayLoader(4, trust_seed=True).load_logs(seeded))
    want = _outcome(lambda: _host(monkeypatch, lambda: GameplayLoader(4, trust_seed=True).load_logs(seeded)))
    assert got == want and got[0] is RuntimeError and "replay job 8 (log 2, player 0)" in got[1], got
    # trust_seed without a seed
    unseeded = [t[0], _with_seed(t[1], None)]
    got = _outcome(lambda: GameplayLoader(4, trust_seed=True).load_logs(unseeded))
    assert got == _outcome(lambda: _host(monkeypatch, lambda: GameplayLoader(4, trust_seed=True).load_logs(unseeded)))
    assert got[0] is ValueError


def test_unreadable_files_raise_the_host_exception(arena_files, tmp_path, monkeypatch):
    """read errors come before any parse error, the first failing file in order raises"""
    from mortal_b200.dataset import GameplayLoader, Grp

    good = arena_files[30:32]
    not_gz = str(tmp_path / "not_gz.json.gz")
    with open(not_gz, "wb") as f:
        f.write(b"this is not gzip")
    not_utf8 = str(tmp_path / "not_utf8.json.gz")
    with gzip.open(not_utf8, "wb") as f:
        f.write(b'{"type":"start_game","names":["\xff","b","c","d"]}\n')
    bad_json = str(tmp_path / "bad_json.json.gz")
    with gzip.open(bad_json, "wb") as f:
        f.write(b"{\n")
    missing = str(tmp_path / "missing.json.gz")
    for files in ([good[0], bad_json, not_gz, good[1]], [good[0], not_utf8, not_gz], [bad_json, missing, good[0]], [good[0], bad_json]):
        for load in (lambda: GameplayLoader(4, oracle=False).load_gz_log_files(files), lambda: Grp.load_gz_log_files(files)):
            got, want = _outcome(load), _outcome(lambda: _host(monkeypatch, load))
            assert isinstance(want, tuple) and got == want, (files, got, want)


def test_grp_on_1024_arena_logs_equals_the_host(arena_files, monkeypatch):
    from mortal_b200.dataset import Grp

    got = Grp.load_gz_log_files(arena_files)
    want = _host(monkeypatch, lambda: Grp.load_gz_log_files(arena_files))
    assert len(got) == len(want) == 1024
    for a, b in zip(got, want):
        _same_grp(a, b)
    assert len({len(g) for g in got}) > 1


def test_grp_runs_on_the_device_libmjx_is_on(arena_files, monkeypatch):
    """a process whose arena or engine initialised libmjx reads its logs on that device, whatever torch's current device is"""
    from mortal_b200 import _lib, _logio
    from mortal_b200.dataset import Grp

    _lib.init(0)
    files = arena_files[40:104]
    want = _host(monkeypatch, lambda: Grp.load_gz_log_files(files))
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 7)  # not a device this process could use
    assert _logio.log_device() == 0
    for a, b in zip(Grp.load_gz_log_files(files), want):
        _same_grp(a, b)


def test_grp_chunks(arena_files, monkeypatch):
    from mortal_b200 import _logio
    from mortal_b200.dataset import Grp

    files = arena_files[:40]
    want = Grp.load_gz_log_files(files)
    for logs, size in ((7, 1 << 30), (4096, 1 << 20)):  # 7 files, or about two arena logs, per chunk
        monkeypatch.setattr(_logio, "CHUNK_LOGS", logs)
        monkeypatch.setattr(_logio, "CHUNK_BYTES", size)
        for a, b in zip(Grp.load_gz_log_files(files), want):
            _same_grp(a, b)


def test_replay_from_device_arrays_checks_the_job_ranges(arena_texts):
    from mortal_b200 import _lib, dataset_codec
    from mortal_b200.env import ReplayEnv

    ev = dataset_codec.parse_log(arena_texts[0])
    jobs = dataset_codec.build_jobs([ev], [[0, 1]])
    dev = torch.device("cuda", 0)
    d = dict(jobs, hdr=torch.from_numpy(jobs["hdr"].view(np.int64)).to(dev), kyoku=torch.from_numpy(jobs["kyoku"].view(np.int64)).to(dev))
    env = ReplayEnv(d, obs_version=4)
    env.close()
    for key, val in (("ev_cnt", len(jobs["hdr"]) + 1), ("ev_off", -1), ("ky_off", len(jobs["kyoku"]) // 19 + 1)):
        bad = dict(d, **{key: np.array([0, val] if key != "ev_cnt" else [len(jobs["hdr"]), val], dtype=np.int32)})
        with pytest.raises(_lib.MjxError, match="lies outside the arrays"):
            ReplayEnv(bad, obs_version=4)
