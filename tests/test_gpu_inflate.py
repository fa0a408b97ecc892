"""mjx_gunzip_dev (k_gunzip, csrc/mjx_inflate.cuh) on the GPU: the corpus of tests/test_emul_inflate.py gets the statuses of the
host emulation and Python's bytes; the CRC-32 equals zlib.crc32 around its lane-chunk boundaries; and the four log readers, over
arena logs mixed with corrupt, truncated, multi-member, zero-padded, non-UTF-8 and plain files, return what the host path returns
and raise what it raises."""
import contextlib
import gzip
import io
import os
import random
import shutil
import zlib

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import inflate_corpus as IC  # noqa: E402


def test_corpus_matches_the_emulation():
    small = [("dynamic", IC.member(IC.deflate(IC.mjai_text(6)), IC.mjai_text(6))),
             ("fixed", IC.member(IC.deflate(b"abcabcabd" * 7, 9, strategy=zlib.Z_FIXED), b"abcabcabd" * 7)),
             ("stored", gzip.compress(b"stored bytes", compresslevel=0, mtime=0))]
    cases = [(n, b, None) for n, b in IC.zlib_corpus()] + IC.handbuilt() + IC.mutations(small)
    blobs = [b for _, b, _ in cases]
    dev, emu = IC.dev_gunzip(blobs), IC.emul_gunzip(blobs)
    for (name, b, want), d, e in zip(cases, dev, emu):
        assert (d is None) == (e is None), name
        if d is not None:
            assert d[0] == e[0], (name, d[0], e[0])
            if d[0] == "OK":
                assert d[1] == e[1], name
        IC.check_contract(name, b, d, want)
    for (name, _), d in zip(IC.zlib_corpus(), dev):
        assert d[0] == "OK", name


def test_crc32_around_chunk_boundaries():
    rng = random.Random(1)
    data = bytes(rng.randrange(256) for _ in range(70000))
    sizes = sorted({0, 1, 31, 32, 33, 65535, 65536, 65537, 70000} | {32 * k + d for k in (1, 2, 3, 31, 32, 33, 1000, 2047) for d in (-1, 0, 1)})
    blobs = [gzip.compress(data[:n], compresslevel=k % 10, mtime=0) for k, n in enumerate(sizes)]
    for n, b, d in zip(sizes, blobs, IC.dev_gunzip(blobs)):
        assert d is not None and d[0] == "OK" and d[1] == data[:n], n
        # the same bytes with the CRC off by one bit: declined for the CRC alone
        bad = bytearray(b); bad[-8] ^= 0x10
        assert IC.dev_gunzip([bytes(bad)])[0][0] == "CRC", n


def test_key_counts_equal_bytes_count():
    from mortal_b200 import _logio
    from mortal_b200.dataset import _AUGMENTED_FIELDS

    keys = [k for k, _ in _AUGMENTED_FIELDS]
    rng = random.Random(4)
    texts = [IC.mjai_text(500, 3), b"", b'"pai"pai"pai"', b'"pai"' * 100]
    texts += [bytes(rng.choice(b'"paiconsumedtehais') for _ in range(rng.randrange(1, 2000))) for _ in range(100)]
    off = np.zeros(len(texts) + 1, dtype=np.int64); np.cumsum([len(t) for t in texts], out=off[1:])
    text = torch.from_numpy(np.frombuffer(b"".join(texts), dtype=np.uint8).copy()).cuda()
    got = _logio.count_keys(text, off, keys, 0)
    for t, row in zip(texts, got):
        assert list(row) == [t.count(k) for k in keys]


# ---- the readers, against the host path ---------------------------------------------------------------------------------------
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

    d = tmp_path_factory.mktemp("inflate_arena")
    torch.manual_seed(5)
    OneVsThree(disable_progress_bar=True, log_dir=str(d)).py_vs_py(_Eng("alpha", 2.0), _Eng("beta", 0.5), (93000, 31), 8)
    files = sorted(os.path.join(d, f) for f in os.listdir(d))
    assert len(files) == 32
    return files


def _variants(src: str):
    """name -> bytes of the file variants made from one arena log"""
    raw = open(src, "rb").read()
    text = gzip.decompress(raw)
    flip = bytearray(raw); flip[len(raw) // 2] ^= 0x40
    return {
        "zero_padded": raw + bytes(16),                        # Python reads it; k_gunzip declines it (TRAILING)
        "level1": gzip.compress(text, compresslevel=1, mtime=0),
        "corrupt": bytes(flip),
        "truncated": raw[:len(raw) // 3],
        "multi_member": raw + raw,
        "non_utf8": gzip.compress(text.replace(b'"alpha"', b'"\xffalpha"', 1), mtime=0),
        "bad_crc": raw[:-8] + bytes([raw[-8] ^ 1]) + raw[-7:],
    }


@pytest.fixture(autouse=True)
def _device_gunzip(monkeypatch):
    """every batch of these tests gunzipped on the device, however few files it has"""
    from mortal_b200 import _logio

    monkeypatch.setattr(_logio, "GZ_DEVICE_MIN_FILES", 0)


def test_small_batches_gunzip_on_the_thread_pool(arena_files, monkeypatch):
    """below GZ_DEVICE_MIN_FILES gzip files the texts are gunzipped on the pool and copied as plain files"""
    from concurrent.futures import ThreadPoolExecutor

    from mortal_b200 import _logio

    monkeypatch.setattr(_logio, "GZ_DEVICE_MIN_FILES", 5)
    items = [_logio.read_gz_file(f) for f in arena_files[:3]] + [(b"not gzip at all", True)]
    with ThreadPoolExecutor(2) as pool:
        T = _logio.stage(items, 0, pool)
        assert T.files == [0, 1, 2] and (T.status.cpu() == 0).all()
        assert T.text.cpu().numpy().tobytes()[:T.log_off[3]] == b"".join(gzip.decompress(r) for r, _ in items[:3])
        # five gzip files: k_gunzip; the 15-byte one is too short to be given to it
        assert _logio.stage(items + [items[0]], 0, pool).files == [0, 1, 2, 4]


def _outcome(fn):
    try:
        return ("ok", fn())
    except Exception as e:  # noqa: BLE001
        return ("raise", type(e), str(e))


def _host(monkeypatch, fn):
    from mortal_b200 import _logio

    with monkeypatch.context() as m:
        m.setattr(_logio, "device_ready", lambda: False)
        return _outcome(fn)


def _dir(tmp_path, name, arena_files, extra):
    d = tmp_path / name
    d.mkdir()
    for f in arena_files[:12]:
        shutil.copy(f, d / os.path.basename(f))
    for fname, data in extra.items():
        (d / fname).write_bytes(data)
    return str(d)


def _mixes(arena_files):
    v = _variants(arena_files[0])
    plain = gzip.decompress(open(arena_files[1], "rb").read())
    good = {"x_zero_padded.json.gz": v["zero_padded"], "x_level1.json.gz": v["level1"], "x_plain.json": plain}
    mixes = {"good": good}
    for bad in ("corrupt", "truncated", "multi_member", "non_utf8", "bad_crc"):
        mixes[bad] = dict(good, **{f"m_{bad}.json.gz": v[bad]})
    return mixes


def test_stat_from_dir_equals_the_host_path(arena_files, tmp_path, monkeypatch):
    from mortal_b200.stat import Stat

    for name, extra in _mixes(arena_files).items():
        d = _dir(tmp_path, name, arena_files, extra)
        got = _outcome(lambda: repr(Stat.from_dir(d, "alpha")))
        want = _host(monkeypatch, lambda: repr(Stat.from_dir(d, "alpha")))
        assert got == want, name


def test_validate_logs_cli_equals_the_host_path(arena_files, tmp_path, monkeypatch):
    from mortal_b200 import _logio, validate_logs

    def run(d):
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            rc = validate_logs.main([d])
        return rc, buf.getvalue()

    def host_run(d):  # the CLI before device gunzip: every file read by _read on the host, then _validate
        import glob

        paths = sorted(set(glob.glob(os.path.join(d, "**", "*.json"), recursive=True))
                       | set(glob.glob(os.path.join(d, "**", "*.json.gz"), recursive=True)))
        verdicts, enc = validate_logs._validate([validate_logs._read(p) for p in paths])
        return 0, "".join(f"\nerror in log {p}\n{validate_logs.message(v, e)}\n" for p, v, e in zip(paths, verdicts, enc)
                          if v is not None)

    mixes = _mixes(arena_files)
    lines = gzip.decompress(open(arena_files[2], "rb").read()).split(b"\n")  # a log that fails to parse at line 6
    lines[5] = lines[5].replace(b'"actor":', b'"actor":9,"y":', 1)
    mixes["parse_error"] = dict(mixes["good"], **{"r_parse_error.json.gz": gzip.compress(b"\n".join(lines), mtime=0)})
    for name, extra in mixes.items():
        d = _dir(tmp_path, name, arena_files, extra)
        assert _outcome(lambda: run(d)) == _outcome(lambda: host_run(d)), name
    assert _logio.device_ready()


def _same_loads(got, want):
    from test_gpu_gameplay_decode import _same, _same_grp

    assert got[0] == want[0]
    if got[0] != "ok":
        assert got == want
        return
    if got[1] and not isinstance(got[1][0], list):  # Grp.load_gz_log_files
        assert len(got[1]) == len(want[1])
        for a, b in zip(got[1], want[1]):
            _same_grp(a, b)
    else:
        _same(got[1], want[1])


@pytest.mark.parametrize("kw", [dict(oracle=False, augmented=True), dict(oracle=False, player_names=["alpha"]),
                                dict(oracle=True, trust_seed=True)], ids=["augmented", "player_names", "oracle_trust_seed"])
def test_gameplay_loader_equals_the_host_path(arena_files, tmp_path, monkeypatch, kw):
    from mortal_b200.dataset import GameplayLoader

    for name, extra in _mixes(arena_files).items():
        d = _dir(tmp_path, name, arena_files, extra)
        files = sorted(os.path.join(d, f) for f in os.listdir(d) if f.endswith(".gz"))
        got = _outcome(lambda: GameplayLoader(4, **kw).load_gz_log_files(files))
        want = _host(monkeypatch, lambda: GameplayLoader(4, **kw).load_gz_log_files(files))
        _same_loads(got, want)


def test_grp_equals_the_host_path(arena_files, tmp_path, monkeypatch):
    from mortal_b200.dataset import Grp

    for name, extra in _mixes(arena_files).items():
        d = _dir(tmp_path, name, arena_files, extra)
        files = sorted(os.path.join(d, f) for f in os.listdir(d) if f.endswith(".gz"))
        _same_loads(_outcome(lambda: Grp.load_gz_log_files(files)), _host(monkeypatch, lambda: Grp.load_gz_log_files(files)))


def test_arena_logs_are_never_declined(arena_files):
    blobs = [open(f, "rb").read() for f in arena_files]
    for f, d in zip(arena_files, IC.dev_gunzip(blobs)):
        assert d[0] == "OK" and d[1] == gzip.decompress(open(f, "rb").read()), f
