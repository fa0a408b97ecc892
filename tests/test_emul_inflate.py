"""k_gunzip's member decode (csrc/mjx_inflate.cuh) in its host build: what it accepts, Python's gzip reads to the same bytes; what
Python rejects, it declines; every stream Python's zlib writes is accepted; hand-built streams for the shapes zlib never writes get
the status the header names; the lane-chunked CRC-32 equals zlib.crc32; the key count equals bytes.count."""
import gzip
import os
import random
import zlib

import numpy as np
import pytest

import emul_lib
import inflate_corpus as IC
from mortal_b200 import _logio


def test_statuses_come_from_the_header():
    assert _logio.GUNZIP_STATUSES == ("ok", "not_gzip", "header", "block", "codes", "symbol", "distance", "truncated", "size", "crc",
                                      "trailing")


def test_every_zlib_stream_is_accepted():
    corpus = IC.zlib_corpus()
    got = IC.emul_gunzip([b for _, b in corpus])
    for (name, b), g in zip(corpus, got):
        assert g is not None and g[0] == "OK", (name, g and g[0])
        IC.check_contract(name, b, g)


def _arena_logs(tmp_path, n=4):
    from mortal_b200 import mjai_log

    nonces = np.arange(4400, 4400 + n, dtype=np.uint64)
    env = emul_lib.EmulEnv(nonces, np.full(n, 2, dtype=np.uint64), enable_quick_eval=True)
    env.enable_log()
    acts = None
    while True:
        env.step(acts)
        if env.num_rows() == 0 and env.num_live() == 0:
            break
        acts = env.policy_test(1)
    words, lens = env.read_log()
    env.close()
    return mjai_log.write_logs(str(tmp_path), words, lens, [(int(x), 2) for x in nonces], [["a", "b", "c", "d"]] * n, "abcd")


def test_arena_logs_are_accepted(tmp_path):
    paths = _arena_logs(tmp_path)
    blobs = [open(p, "rb").read() for p in paths]
    for p, b, g in zip(paths, blobs, IC.emul_gunzip(blobs)):
        assert g[0] == "OK" and g[1] == gzip.open(p, "rb").read(), p


@pytest.mark.parametrize("name", [n for n, _, _ in IC.handbuilt()])
def test_handbuilt_streams(name):
    case = {n: (b, w) for n, b, w in IC.handbuilt()}[name]
    b, want = case
    IC.check_contract(name, b, IC.emul_gunzip([b])[0], want)


def test_python_agrees_on_the_handbuilt_streams_it_accepts():
    """the single-distance-code and literal-only shapes are legal: zlib reads them, and so does the device"""
    for name, b, want in IC.handbuilt():
        if want == "OK":
            assert IC.python_gunzip(b) is not None, name


def test_mutations():
    small = [("dynamic", IC.member(IC.deflate(IC.mjai_text(6)), IC.mjai_text(6))),
             ("fixed", IC.member(IC.deflate(b"abcabcabd" * 7, 9, strategy=zlib.Z_FIXED), b"abcabcabd" * 7)),
             ("stored", gzip.compress(b"stored bytes", compresslevel=0, mtime=0))]
    cases = IC.mutations(small)
    got = IC.emul_gunzip([b for _, b, _ in cases])
    for (name, b, want), g in zip(cases, got):
        IC.check_contract(name, b, g, want)
    # a member followed by anything is declined, whatever Python makes of it
    for (name, b, _), g in zip(cases, got):
        if name.endswith(("zero-padding", "second-member", "garbage")):
            assert g is None or g[0] != "OK", name


def test_crc32_at_chunk_boundaries():
    rng = random.Random(3)
    data = bytes(rng.randrange(256) for _ in range(5000))
    for n in sorted({0, 1, 2, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025, 4095, 4096, 4097, 5000} | {32 * k + d for k in range(1, 20) for d in (-1, 0, 1)}):
        buf = np.frombuffer(data[:n] or b"\0", dtype=np.uint8)
        assert emul_lib.lib().emulz_crc32(buf.ctypes.data, n) == zlib.crc32(data[:n]), n


def _count(texts, keys):
    off = np.zeros(len(texts) + 1, dtype=np.int64); np.cumsum([len(t) for t in texts], out=off[1:])
    text = np.frombuffer(b"".join(texts) or b"\0", dtype=np.uint8)
    koff = np.zeros(len(keys) + 1, dtype=np.int32); np.cumsum([len(k) for k in keys], out=koff[1:])
    kb = np.frombuffer(b"".join(keys), dtype=np.uint8)
    out = np.zeros((len(texts), len(keys)), dtype=np.int64)
    assert emul_lib.lib().emulz_count_keys(len(texts), text.ctypes.data, int(off[-1]), off.ctypes.data, kb.ctypes.data, koff.ctypes.data,
                                           len(keys), out.ctypes.data) == 0
    return out


def test_key_count_is_bytes_count():
    from mortal_b200.dataset import _AUGMENTED_FIELDS

    keys = [k for k, _ in _AUGMENTED_FIELDS]
    rng = random.Random(9)
    texts = [b"", b'"pai"', b'"pai"pai"', b'"pai"pai"pai"', b'x"pai"' * 40, b'"pai""pai"', b"aaaa", IC.mjai_text(300, 2)]
    texts += [bytes(rng.choice(b'"paiconsumed') for _ in range(rng.randrange(1, 300))) for _ in range(50)]
    got = _count(texts, keys)
    for t, row in zip(texts, got):
        assert list(row) == [t.count(k) for k in keys], t
    # self-overlapping keys: counted left to right without overlap
    assert list(_count([b"aaaaa", b"abababa"], [b"aa", b"aba", b"a"])[0]) == [2, 0, 5]
    assert list(_count([b"aaaaa", b"abababa"], [b"aa", b"aba", b"a"])[1]) == [0, 2, 4]


def test_readers_size_and_route_files():
    ok = gzip.compress(b"x" * 100)
    assert _logio.gz_isize(ok) == 100
    assert _logio.gz_isize(ok[:17]) is None  # shorter than a header and a trailer
    assert _logio.gz_isize(ok[:-4] + (1032 * len(ok) + 1).to_bytes(4, "little")) is None  # no deflate stream expands that far
    assert _logio.text_size((ok, True)) == 100 and _logio.text_size((b"abc", False)) == 3 and _logio.text_size((None, True)) == 0


def test_read_file(tmp_path):
    p = tmp_path / "a.json.gz"
    p.write_bytes(b"raw")
    assert _logio.read_file(str(p)) == (b"raw", True) and _logio.read_gz_file(str(p)) == (b"raw", True)
    assert _logio.read_file(str(tmp_path / "missing.json")) == (None, False)


def test_golden_fixture_round_trip():
    path = os.path.join(IC.ROOT, "tests", "golden", "reference_engine_game.json.gz")
    b = open(path, "rb").read()
    g = IC.emul_gunzip([b])[0]
    assert g[0] == "OK" and g[1] == gzip.decompress(b)


def test_sanitized_run():
    """tests/sanitized_inflate_run.py: the hostile inputs under AddressSanitizer + UBSan"""
    import subprocess
    import sys

    libs = [subprocess.run(["gcc", f"-print-file-name={n}"], capture_output=True, text=True).stdout.strip()
            for n in ("libasan.so", "libubsan.so")]
    if not all(os.path.isabs(p) and os.path.exists(p) for p in libs):
        pytest.skip("gcc's ASan / UBSan runtimes are not installed")
    env = dict(os.environ, LD_PRELOAD=":".join(libs), ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([sys.executable, os.path.join(IC.ROOT, "tests", "sanitized_inflate_run.py")], env=env, capture_output=True,
                       text=True, timeout=1800)
    assert r.returncode == 0 and "sanitised gunzip run finished" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
