"""Stat.from_dir on the GPU (k_mjai_decode with the deltas output + k_stat_logs): on 1,024 arena logs it equals the host path
for every engine name and for a name that appears nowhere; per log the kernel equals Stat.from_game on format variations and
mutated logs, and hostile files give the host path's result or exception type; the deltas fill writes the plain fill's arrays plus
the json deltas; chunking and file order do not matter; a mixed directory gives the host result; the CLI prints the reference
report of the host Stat."""
import gzip
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import log_mutations as LM
import mjai_lib as M
import stat_lib as S

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Eng:
    engine_type, version, is_oracle, enable_quick_eval, enable_rule_based_agari_guard = "mortal", 4, False, True, False

    def __init__(self, name, bias):
        self.name, self.bias = name, bias

    def react_device(self, obs, masks):
        q = torch.rand(masks.shape, device=masks.device)
        q[:, :34] += self.bias * obs[:, 876, :] + obs[:, 875, :]
        q = q.masked_fill(~masks, -1.0)
        return q.argmax(-1), q


def _host(paths, name):
    """today's from_dir over `paths`: every file through the host code"""
    from mortal_b200.stat import Stat, _host_log_stat

    total = Stat()
    for p in paths:
        total = total + _host_log_stat(p, name)
    return total


def _same(a, b):
    from mortal_b200.stat import COUNTERS

    return all(getattr(a, c) == getattr(b, c) for c in COUNTERS)


def _outcome(fn):
    try:
        return fn()
    except Exception as e:  # noqa: BLE001
        return type(e)


@pytest.fixture(scope="module")
def arena_dir(tmp_path_factory):
    from mortal_b200.libriichi.arena import OneVsThree

    d = tmp_path_factory.mktemp("arena_stat")
    OneVsThree(disable_progress_bar=True, log_dir=str(d)).py_vs_py(_Eng("alpha", 2.0), _Eng("beta", 0.5), (83000, 17), 256)
    return d


@pytest.fixture(scope="module")
def arena_texts(arena_dir):
    return [gzip.open(os.path.join(arena_dir, f), "rt").read() for f in sorted(os.listdir(arena_dir))]


def test_device_path_is_taken():
    from mortal_b200.stat import _device_ready

    assert _device_ready()


def test_from_dir_equals_the_host_path_on_arena_logs(arena_dir):
    from mortal_b200.stat import Stat, _log_paths

    paths = _log_paths(str(arena_dir))
    assert len(paths) == 1024
    got = {n: Stat.from_dir(str(arena_dir), n) for n in ("alpha", "beta", "nobody")}
    for n, st in got.items():
        assert _same(st, _host(paths, n)), n
    assert got["alpha"].game + got["beta"].game == 4096 and got["alpha"].game == 1024 and got["nobody"].game == 0
    assert got["alpha"].agari > 0 and got["beta"].houjuu > 0


def test_arena_logs_are_counted_on_the_device(arena_dir, monkeypatch):
    """with the host reader disabled, from_dir still returns the host result: every arena log was counted by k_stat_logs"""
    from mortal_b200 import stat

    paths = stat._log_paths(str(arena_dir))
    want = {n: _host(paths, n) for n in ("alpha", "nobody")}

    def no_host(path, name):
        raise AssertionError(f"{path} went to the host path")

    monkeypatch.setattr(stat, "_host_log_stat", no_host)
    for n, w in want.items():
        assert _same(stat.Stat.from_dir(str(arena_dir), n), w), n


def test_from_dir_uses_the_device_libmjx_is_on(arena_dir, monkeypatch):
    """a process whose arena or engine initialised libmjx counts on that device, whatever torch's current device is"""
    from mortal_b200 import _lib, stat

    _lib.init(0)
    paths = stat._log_paths(str(arena_dir))[:64]
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 7)  # not a device this process could use
    assert stat._stat_device() == 0
    assert _same(stat._device_from_dir(paths, "alpha"), _host(paths, "alpha"))


def _kernel_rows(blobs, masks):
    """decode_dev(deltas=True) + mjx_stat_logs_dev over the given seat masks -> (accept, int64 [n, 44], int32 [n])"""
    from mortal_b200 import _lib
    from mortal_b200.validate_logs import decode_dev

    L = _lib.load()
    D = decode_dev(blobs, 0, deltas=True)
    n = len(blobs)
    out = torch.empty((n, len(S.NAMES)), dtype=torch.int64, device="cuda")
    status = torch.empty(n, dtype=torch.int32, device="cuda")
    seats = torch.tensor(np.asarray(masks, dtype=np.uint8), device="cuda")
    ptr = lambda t: t.data_ptr() if t.numel() else None
    _lib.check(L.mjx_stat_logs_dev(n, ptr(D.hdr), D.offs[0].data_ptr(), D.offs[1].data_ptr(), D.hdr.numel(), ptr(D.kyoku),
                                   D.offs[2].data_ptr(), D.kyoku.numel(), ptr(D.deltas), ptr(D.has_deltas), seats.data_ptr(),
                                   out.data_ptr(), status.data_ptr(), torch.cuda.current_stream().cuda_stream), "mjx_stat_logs_dev")
    return D.accept, out.cpu().numpy(), status.cpu().numpy()


def _per_log(texts, masks_of, want_accepted=False):
    blobs = [t.encode("utf-8") for t in texts]
    events = [[json.loads(x) for x in t.splitlines() if x.strip()] for t in texts]
    counted = flagged = 0
    for m_fixed in (None, 15):
        masks = [m_fixed if m_fixed is not None else masks_of(ev) for ev in events]
        accept, out, status = _kernel_rows(blobs, masks)
        if want_accepted:
            assert accept.all()
        for i, ev in enumerate(events):
            if not accept[i]:
                continue
            want = S.host_row(ev, masks[i])
            if want is None:
                assert status[i] != 0 and not out[i].any(), i
                flagged += 1
            else:
                assert status[i] == 0 and np.array_equal(out[i], want), (i, masks[i])
                counted += 1
    return counted, flagged


def test_format_variations_per_log(arena_texts):
    rng = np.random.default_rng(47)
    texts = [M.vary([json.loads(x) for x in t.splitlines()], rng) for t in arena_texts[:128]]
    counted, _ = _per_log(texts, lambda ev: S.seat_mask(ev, "café"), want_accepted=True)
    assert counted == 256


def test_mutation_corpus_per_log(arena_texts):
    games = [[json.loads(x) for x in t.splitlines()] for t in arena_texts[:64]]
    texts = []
    for _, t in LM.mutated_corpus(games, 20, np.random.default_rng(53)):
        try:
            [json.loads(x) for x in t.splitlines() if x.strip()]
            texts.append(t)
        except ValueError:
            pass
    counted, flagged = _per_log(texts, lambda ev: S.seat_mask(ev, "alpha"))
    assert counted > len(texts) and flagged > 0  # hora_field_removed without deltas is flagged for the selected seats


def test_hostile_files_give_the_host_result_or_exception(arena_texts, tmp_path):
    from mortal_b200.stat import _device_from_dir, _host_log_stat

    rng = np.random.default_rng(59)
    paths = []
    for k, (_, b) in enumerate(M.hostile_corpus(arena_texts[:32], 12, rng)):
        p = tmp_path / (f"h{k}.json.gz" if k % 2 else f"h{k}.json")
        p.write_bytes(gzip.compress(b) if k % 2 else b)
        paths.append(str(p))
    raised = 0
    for p in paths:
        want = _outcome(lambda: _host_log_stat(p, "alpha"))
        got = _outcome(lambda: _device_from_dir([p], "alpha"))
        if isinstance(want, type):
            assert got is want, p
            raised += 1
        else:
            assert not isinstance(got, type) and _same(got, want), p
    assert raised > 0
    # all together, in one chunk: the first failing file's exception type
    outcomes = [_outcome(lambda: _host_log_stat(p, "alpha")) for p in paths]
    first = next(o for o in outcomes if isinstance(o, type))
    assert _outcome(lambda: _device_from_dir(paths, "alpha")) is first


def test_deltas_fill_matches_the_plain_fill(arena_texts):
    from mortal_b200.validate_logs import decode_dev

    blobs = [t.encode("utf-8") for t in arena_texts]
    A, B = decode_dev(blobs), decode_dev(blobs, deltas=True)
    assert A.accept.all() and np.array_equal(A.counts, B.counts)
    for k in ("hdr", "lines", "kyoku", "hora"):
        assert torch.equal(getattr(A, k), getattr(B, k)), k
    d, has = B.deltas.cpu().numpy(), B.has_deltas.cpu().numpy()
    n = 0
    for i, t in enumerate(arena_texts):
        events = [json.loads(x) for x in t.splitlines() if x.strip()]
        for k, ev in enumerate(events):
            if ev["type"] in ("hora", "ryukyoku"):
                e = int(B.ev_off[i]) + k
                assert has[e] == 1 and list(d[e]) == ev["deltas"], (i, k)
                n += 1
    assert n > 1024


def test_chunking_and_file_order_do_not_matter(arena_dir, monkeypatch):
    from mortal_b200 import stat

    paths = stat._log_paths(str(arena_dir))[:200]
    full = stat._device_from_dir(paths, "alpha")
    assert _same(full, _host(paths, "alpha"))
    monkeypatch.setattr(stat, "CHUNK_LOGS", 7)
    perm = [paths[i] for i in np.random.default_rng(61).permutation(len(paths))]
    assert _same(stat._device_from_dir(perm, "alpha"), full)
    monkeypatch.setattr(stat, "CHUNK_LOGS", 4096)
    monkeypatch.setattr(stat, "CHUNK_BYTES", 3 << 20)  # a few arena logs per chunk
    assert _same(stat._device_from_dir(perm, "alpha"), full)
    assert _same(stat._device_from_dir(paths[:1], "alpha"), _host(paths[:1], "alpha"))


def _mixed_dir(d, arena_texts):
    events = [json.loads(x) for x in arena_texts[5].splitlines()]
    events[0]["names"] = ["p", "q", "r", "s"]  # the player is not in it, so missing deltas are no error
    for ev in events:
        if ev["type"] in ("hora", "ryukyoku"):
            ev.pop("deltas")
    layout = {"a/one.json": arena_texts[0], "a/b/two.json.gz": arena_texts[1], "three.json.gz": arena_texts[2],
              "crlf.json": arena_texts[3].replace("\n", "\r\n"), "lone_cr.json": arena_texts[4].replace("\n", "\r", 3),
              "no_deltas.json": "\n".join(json.dumps(e) for e in events) + "\n"}
    for name, text in layout.items():
        p = d / name
        p.parent.mkdir(parents=True, exist_ok=True)
        if name.endswith(".gz"):
            with gzip.open(p, "wt", newline="") as f:
                f.write(text)
        else:
            p.write_bytes(text.encode("utf-8"))
    return d


def test_mixed_directory(arena_texts, tmp_path):
    from mortal_b200.stat import Stat, _log_paths
    from mortal_b200.validate_logs import decode_dev

    d = _mixed_dir(tmp_path, arena_texts)
    assert not decode_dev([(d / "lone_cr.json").read_bytes()]).accept[0]  # declined: read on the host
    paths = _log_paths(str(d))
    assert len(paths) == 6
    for n in ("alpha", "beta", "nobody"):
        assert _same(Stat.from_dir(str(d), n), _host(paths, n)), n
    (d / "a" / "notgz.json.gz").write_bytes(b"plain text, not gzip")
    want = _outcome(lambda: _host(_log_paths(str(d)), "alpha"))
    assert isinstance(want, type) and _outcome(lambda: Stat.from_dir(str(d), "alpha")) is want


def test_cli(arena_texts, tmp_path):
    from mortal_b200.stat import _log_paths

    d = _mixed_dir(tmp_path / "ok", arena_texts)
    want = _host(_log_paths(str(d)), "alpha").reference_text() + "\n"
    r = subprocess.run([sys.executable, "-m", "mortal_b200.stat", str(d), "alpha"], cwd=ROOT, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr
    assert r.stdout == want
    (d / "notgz.json.gz").write_bytes(b"plain text, not gzip")
    r = subprocess.run([sys.executable, "-m", "mortal_b200.stat", str(d), "alpha"], cwd=ROOT, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 1 and r.stdout == "" and "Error" in r.stderr
    r = subprocess.run([sys.executable, "-m", "mortal_b200.stat", str(d)], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 2 and r.stdout == ""
