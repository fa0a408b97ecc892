#!/usr/bin/env python
"""Runs the gzip member decode and the key count (csrc/mjx_inflate.cuh, host build) under AddressSanitizer + UBSan over the zlib
corpus, the hand-built streams, every mutation of a few small streams and random bytes behind a gzip header: every status must
keep the contract (OK => gzip.decompress's bytes), and no read or write may leave its buffer. Each file is packed into a buffer
of its own exact size, so a read past a file's end is a read past the allocation. Usage (tests/test_emul_inflate.py runs it):

    LD_PRELOAD=$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so) ASAN_OPTIONS=detect_leaks=0 \\
        python tests/sanitized_inflate_run.py
"""
import gzip
import os
import random
import sys
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import emul_lib as E  # noqa: E402

L = E.lib(sanitize=True)
import inflate_corpus as IC  # noqa: E402
from mortal_b200 import _logio  # noqa: E402


def one(b: bytes):
    """one file in buffers of its exact sizes (no slack for a stray read to land in)"""
    n = _logio.gz_isize(b)
    if n is None:
        return None
    gz = np.frombuffer(b, dtype=np.uint8).copy()
    out = np.empty(n, dtype=np.uint8) if n else np.empty(1, dtype=np.uint8)[:0]
    gz_off = np.array([0, len(b)], dtype=np.int64)
    out_off = np.array([0, n], dtype=np.int64)
    st = np.zeros(1, dtype=np.int32)
    assert L.emulz_gunzip(1, gz.ctypes.data, len(b), gz_off.ctypes.data, out.ctypes.data if n else gz.ctypes.data, n,
                          out_off.ctypes.data, st.ctypes.data) == 0
    return _logio.GUNZIP_STATUSES[st[0]].upper(), out.tobytes()


counts = {}
cases = [(n, b, None) for n, b in IC.zlib_corpus()] + IC.handbuilt()
small = [("dynamic", IC.member(IC.deflate(IC.mjai_text(6)), IC.mjai_text(6))),
         ("fixed", IC.member(IC.deflate(b"abcabcabd" * 7, 9, strategy=zlib.Z_FIXED), b"abcabcabd" * 7)),
         ("stored", gzip.compress(b"stored bytes", compresslevel=0, mtime=0))]
cases += IC.mutations(small)
rng = random.Random(17)
head = bytes([0x1F, 0x8B, 8, 0, 0, 0, 0, 0, 0, 255])
for k in range(2000):  # random deflate bits, with a trailer whose ISIZE is small enough to be taken
    body = bytes(rng.randrange(256) for _ in range(rng.randrange(1, 200)))
    cases.append((f"random{k}", head + body + bytes(4) + rng.randrange(0, 2000).to_bytes(4, "little"), None))
for name, b, want in cases:
    g = one(b)
    IC.check_contract(name, b, g, want)
    if g is not None:
        counts[g[0]] = counts.get(g[0], 0) + 1
rng = np.random.default_rng(5)
keys = [k for k, _ in __import__("mortal_b200.dataset", fromlist=["_AUGMENTED_FIELDS"])._AUGMENTED_FIELDS]
koff = np.zeros(len(keys) + 1, dtype=np.int32); np.cumsum([len(k) for k in keys], out=koff[1:])
kb = np.frombuffer(b"".join(keys), dtype=np.uint8).copy()
for t in range(300):
    text = bytes(rng.choice(np.frombuffer(b'"paitehisconsumed', dtype=np.uint8), size=int(rng.integers(1, 400))))
    buf = np.frombuffer(text, dtype=np.uint8).copy()
    off = np.array([0, len(text)], dtype=np.int64)
    out = np.zeros(len(keys), dtype=np.int64)
    assert L.emulz_count_keys(1, buf.ctypes.data, len(text), off.ctypes.data, kb.ctypes.data, koff.ctypes.data, len(keys),
                              out.ctypes.data) == 0
    assert list(out) == [text.count(k) for k in keys], text
print(f"sanitised gunzip run finished: {len(cases)} files, statuses {dict(sorted(counts.items()))}; 300 key counts equal bytes.count")
