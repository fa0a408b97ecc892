"""The inputs of the device gunzip tests (tests/test_emul_inflate.py, tests/sanitized_inflate_run.py, tests/test_gpu_inflate.py):
gzip members from Python's zlib at every setting the tests name, hand-built DEFLATE streams for the shapes zlib never writes, and
mutations; plus the two ways of running them (the host emulation and mjx_gunzip_dev), both sized as the readers size a slot."""
import gzip
import os
import random
import struct
import zlib

import numpy as np

from mortal_b200 import _logio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATUS = {name.upper(): k for k, name in enumerate(_logio.GUNZIP_STATUSES)}
STRATEGIES = {"default": zlib.Z_DEFAULT_STRATEGY, "filtered": zlib.Z_FILTERED, "huffman_only": zlib.Z_HUFFMAN_ONLY,
              "rle": zlib.Z_RLE, "fixed": zlib.Z_FIXED}


def member(deflate: bytes, data: bytes, flags: int = 0, name: bytes = b"", comment: bytes = b"", extra: bytes = b"") -> bytes:
    """a gzip member around a raw deflate stream of `data`, with the optional header fields of `flags` (RFC 1952)"""
    head = bytes([0x1F, 0x8B, 8, flags]) + struct.pack("<I", 12345) + bytes([2, 255])
    if flags & 4:
        head += struct.pack("<H", len(extra)) + extra
    if flags & 8:
        head += name + b"\0"
    if flags & 16:
        head += comment + b"\0"
    if flags & 2:
        head += struct.pack("<H", zlib.crc32(head) & 0xFFFF)
    return head + deflate + struct.pack("<II", zlib.crc32(data), len(data) & 0xFFFFFFFF)


def deflate(data: bytes, level=9, wbits=15, mem=8, strategy=zlib.Z_DEFAULT_STRATEGY, flushes=()) -> bytes:
    """zlib's raw deflate of data, with flush(mode) after every piece when `flushes` names the modes between pieces"""
    c = zlib.compressobj(level, zlib.DEFLATED, -wbits, mem, strategy)
    if not flushes:
        return c.compress(data) + c.flush()
    out, step = [], max(1, len(data) // (len(flushes) + 1))
    for k, mode in enumerate(flushes):
        out += [c.compress(data[k * step:(k + 1) * step]), c.flush(mode)]
    return b"".join(out) + c.compress(data[len(flushes) * step:]) + c.flush()


def mjai_text(n_lines=400, seed=0) -> bytes:
    """text shaped like an mjai log (JSON lines with repeated keys and tile names)"""
    rng = random.Random(seed)
    tiles = [f"{k}{s}" for s in "mps" for k in range(1, 10)] + ["E", "S", "W", "N", "P", "F", "C", "5mr"]
    lines = ['{"type":"start_game","names":["a","b","c","d"],"seed":[1,2]}']
    for _ in range(n_lines):
        ty = rng.choice(["tsumo", "dahai"])
        lines.append(f'{{"type":"{ty}","actor":{rng.randrange(4)},"pai":"{rng.choice(tiles)}"'
                     + (f',"tsumogiri":{rng.choice(["true", "false"])}}}' if ty == "dahai" else "}"))
    return ("\n".join(lines) + "\n").encode()


def payloads():
    rng = random.Random(7)
    return {
        "mjai": mjai_text(),
        "random": bytes(rng.randrange(256) for _ in range(20000)),
        "run": b"a" * 100000,
        "mixed": mjai_text(200, 1) + bytes(rng.randrange(256) for _ in range(3000)) + b"xyz" * 5000,
    }


def zlib_corpus():
    """(name, gz bytes) that Python's zlib writes: every level, strategy, wbits 9-15 and memLevel 1 / 9, mid-stream flushes,
    edge sizes, header fields, the golden fixture"""
    P = payloads()
    out = []
    for level in range(10):
        for sname, strat in STRATEGIES.items():
            for wbits in range(9, 16):
                for mem in (1, 9):
                    key = ("mjai", "random", "run", "mixed")[(level + wbits + mem) % 4]
                    out.append((f"l{level}-{sname}-w{wbits}-m{mem}-{key}", member(deflate(P[key], level, wbits, mem, strat), P[key])))
    for mode_name, mode in (("sync", zlib.Z_SYNC_FLUSH), ("full", zlib.Z_FULL_FLUSH), ("partial", zlib.Z_PARTIAL_FLUSH),
                            ("block", zlib.Z_BLOCK)):
        for level in (1, 6, 9):
            d = P["mixed"]
            out.append((f"flush-{mode_name}-l{level}", member(deflate(d, level, flushes=[mode] * 5), d)))
    for name, d in (("empty", b""), ("one", b"x"), ("stored-65535", bytes(range(256)) * 255 + bytes(255)),
                    ("stored-0", b"")):
        level = 0 if name.startswith("stored") else 9
        out.append((name, member(deflate(d, level), d)))
        out.append((name + "-gzip", gzip.compress(d, compresslevel=level, mtime=0)))
    d = P["mjai"]
    for flags, kw in ((8, dict(name=b"log.json")), (16, dict(comment=b"a comment")), (4, dict(extra=b"AB\x04\x00wxyz")),
                      (2, {}), (30, dict(name=b"n", comment=b"c", extra=b"x"))):
        out.append((f"header-{flags}", member(deflate(d), d, flags, **kw)))
    with open(os.path.join(ROOT, "tests", "golden", "reference_engine_game.json.gz"), "rb") as f:
        out.append(("golden", f.read()))
    return out


# ---- hand-built streams -------------------------------------------------------------------------------------------------------
class BitWriter:
    def __init__(self):
        self.bits = []

    def put(self, v: int, n: int):  # n bits of v, LSB first (header fields, extra bits)
        self.bits += [(v >> k) & 1 for k in range(n)]

    def code(self, c: int, n: int):  # a Huffman code, MSB first
        self.bits += [(c >> (n - 1 - k)) & 1 for k in range(n)]

    def align(self):
        self.bits += [0] * (-len(self.bits) % 8)

    def raw(self, b: bytes):
        self.align()
        for x in b:
            self.put(x, 8)

    def bytes(self) -> bytes:
        self.align()
        return bytes(sum(self.bits[i + k] << k for k in range(8)) for i in range(0, len(self.bits), 8))


def canonical(lens):
    """symbol -> (code, length) of the canonical code with these lengths (RFC 1951 3.2.2)"""
    count = [0] * 16
    for n in lens:
        count[n] += 1
    count[0] = 0
    nxt, code = [0] * 16, 0
    for n in range(1, 16):
        code = (code + count[n - 1]) << 1
        nxt[n] = code
    out = {}
    for s, n in enumerate(lens):
        if n:
            out[s] = (nxt[n], n); nxt[n] += 1
    return out


def fixed_lit(w: BitWriter, s: int):
    if s < 144:
        w.code(0x30 + s, 8)
    elif s < 256:
        w.code(0x190 + s - 144, 9)
    elif s < 280:
        w.code(s - 256, 7)
    else:
        w.code(0xC0 + s - 280, 8)


def dynamic_header(w: BitWriter, lit, dist, final=1, cl=None, hlit=None, hdist=None, seq=None):
    """a dynamic block header: lengths `lit` / `dist` sent as plain code-length symbols (or the symbols `seq`: (sym, extra
    bits, extra value)), over the code-length code `cl` (default: a complete code of all 19 symbols)"""
    cl = (cl if cl is not None else [4] * 13 + [5] * 6) + [0] * 19
    cl = cl[:19]
    w.put(final, 1); w.put(2, 2)
    w.put((hlit if hlit is not None else len(lit)) - 257, 5)
    w.put((hdist if hdist is not None else len(dist)) - 1, 5)
    order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
    w.put(19 - 4, 4)
    for s in order:
        w.put(cl[s], 3)
    cc = canonical(cl)
    for sym, nb, v in (seq if seq is not None else [(n, 0, 0) for n in list(lit) + list(dist)]):
        w.code(*cc[sym])
        if nb:
            w.put(v, nb)
    return canonical(lit), canonical(dist)


_LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
_LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
_DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
              8193, 12289, 16385, 24577]
_DIST_EXTRA = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]


def length_sym(n):
    s = max(k for k in range(29) if _LEN_BASE[k] <= n and (k < 28 or n == 258))
    return 257 + s, _LEN_EXTRA[s], n - _LEN_BASE[s]


def dist_sym(d):
    s = max(k for k in range(30) if _DIST_BASE[k] <= d)
    return s, _DIST_EXTRA[s], d - _DIST_BASE[s]


def handbuilt():
    """(name, gz bytes, the status the device must give); the member's trailer is that of `data`, the intended output"""
    out = []

    def add(name, w, data, want):
        out.append((name, member(w.bytes(), data), want))

    # a single distance code of length 1 (zlib accepts it): 'a', then a length-3 match at distance 1
    lit = [0] * 257 + [2]; lit[97] = 1; lit[256] = 2
    w = BitWriter(); L, D = dynamic_header(w, lit, [1])
    w.code(*L[97]); w.code(*L[257]); w.code(*D[0]); w.code(*L[256])
    add("single-distance-code", w, b"aaaa", "OK")
    # the same code with the other bit pattern, which no distance code has
    w = BitWriter(); L, D = dynamic_header(w, lit, [1])
    w.code(*L[97]); w.code(*L[257]); w.code(1, 1); w.code(*L[256])
    add("single-distance-code-bad-pattern", w, b"aaaa", "SYMBOL")
    # no distance codes: a literal-only block (zlib accepts it); a length symbol in it has no distance to read
    lit2 = [0] * 257; lit2[97] = 1; lit2[256] = 1
    w = BitWriter(); L, _ = dynamic_header(w, lit2, [0])
    w.code(*L[97]); w.code(*L[97]); w.code(*L[256])
    add("no-distance-codes", w, b"aa", "OK")
    lit3 = [0] * 258; lit3[97] = 1; lit3[256] = 2; lit3[257] = 2
    w = BitWriter(); L, _ = dynamic_header(w, lit3, [0])
    w.code(*L[97]); w.code(*L[257]); w.code(*L[256])
    add("no-distance-codes-length", w, b"aaaa", "SYMBOL")
    # code sets
    w = BitWriter(); dynamic_header(w, [1] * 3 + [0] * 253 + [1], [1, 1])
    add("lit-over-subscribed", w, b"", "CODES")
    w = BitWriter(); dynamic_header(w, [2] * 2 + [0] * 254 + [2], [1, 1])
    add("lit-incomplete", w, b"", "CODES")
    w = BitWriter(); L, _ = dynamic_header(w, [0] * 256 + [1], [1, 1])
    w.code(*L[256])
    add("lit-single-code", w, b"", "CODES")  # zlib accepts a lone length-1 code here; the device declines it
    w = BitWriter(); dynamic_header(w, lit, [1, 1, 1])
    add("dist-over-subscribed", w, b"", "CODES")
    w = BitWriter(); dynamic_header(w, lit, [2, 2, 2])
    add("dist-incomplete", w, b"", "CODES")
    w = BitWriter(); dynamic_header(w, lit, [2])
    add("dist-single-code-length-2", w, b"", "CODES")
    w = BitWriter(); dynamic_header(w, [1] * 2 + [0] * 255, [1, 1])
    add("no-end-of-block", w, b"", "CODES")
    w = BitWriter(); dynamic_header(w, lit, [1, 1], hlit=287, seq=[])
    add("hlit-287", w, b"", "CODES")
    w = BitWriter(); dynamic_header(w, lit, [1, 1], hdist=31, seq=[])
    add("hdist-31", w, b"", "CODES")
    w = BitWriter(); dynamic_header(w, lit, [1, 1], seq=[(16, 2, 0)])
    add("repeat-first", w, b"", "CODES")
    w = BitWriter(); dynamic_header(w, lit, [1, 1], seq=[(18, 7, 127)] * 2 + [(18, 7, 127)])
    add("repeat-past-count", w, b"", "CODES")
    w = BitWriter(); dynamic_header(w, lit, [1], cl=[1, 1, 1] + [0] * 16, seq=[])
    add("cl-over-subscribed", w, b"", "CODES")
    w = BitWriter(); dynamic_header(w, lit, [1], cl=[2, 2] + [0] * 17, seq=[])
    add("cl-incomplete", w, b"", "CODES")
    w = BitWriter(); dynamic_header(w, lit, [1], cl=[1] + [0] * 18, seq=[])
    add("cl-single-code", w, b"", "CODES")
    # fixed-code symbols no table has
    for s, name in ((286, "length-286"), (287, "length-287")):
        w = BitWriter(); w.put(1, 1); w.put(1, 2); fixed_lit(w, 97); fixed_lit(w, s); w.code(0, 5); fixed_lit(w, 256)
        add(name, w, b"aaaa", "SYMBOL")
    for d in (30, 31):
        w = BitWriter(); w.put(1, 1); w.put(1, 2); fixed_lit(w, 97); fixed_lit(w, 257); w.code(d, 5); fixed_lit(w, 256)
        add(f"distance-{d}", w, b"aaaa", "SYMBOL")
    # blocks
    w = BitWriter(); w.put(1, 1); w.put(3, 2)
    add("block-type-3", w, b"", "BLOCK")
    w = BitWriter(); w.put(1, 1); w.put(0, 2); w.align(); w.put(3, 16); w.put(0, 16); w.raw(b"abc")
    add("stored-nlen", w, b"abc", "BLOCK")
    # a distance back past the start
    w = BitWriter(); w.put(1, 1); w.put(1, 2); fixed_lit(w, 97); fixed_lit(w, 257); w.code(1, 5); fixed_lit(w, 256)
    add("distance-past-start", w, b"aaaa", "DISTANCE")
    # length 258 at distance 32768 (zlib never reaches that far back): 32768 stored bytes, then the match twice
    rng = random.Random(5)
    head = bytes(rng.randrange(256) for _ in range(32768))
    w = BitWriter(); w.put(0, 1); w.put(0, 2); w.align(); w.put(32768, 16); w.put(32768 ^ 0xFFFF, 16); w.raw(head)
    w.put(1, 1); w.put(1, 2)
    data = bytearray(head)
    for _ in range(2):
        s, nb, v = length_sym(258); fixed_lit(w, s); w.put(v, nb)
        ds, dnb, dv = dist_sym(32768); w.code(ds, 5); w.put(dv, dnb)
        for _ in range(258):
            data.append(data[-32768])
    fixed_lit(w, 256)
    add("length-258-distance-32768", w, bytes(data), "OK")
    # stored blocks of 0 and 65,535 bytes
    w = BitWriter(); w.put(0, 1); w.put(0, 2); w.align(); w.put(0, 16); w.put(0xFFFF, 16)
    w.put(1, 1); w.put(0, 2); w.align(); w.put(65535, 16); w.put(0, 16); w.raw(bytes(range(256)) * 255 + bytes(255))
    add("stored-0-and-65535", w, bytes(range(256)) * 255 + bytes(255), "OK")
    # distance-1 overlapping copies of every length
    w = BitWriter(); w.put(1, 1); w.put(1, 2); fixed_lit(w, 120)
    data = bytearray(b"x")
    for n in range(3, 259):
        s, nb, v = length_sym(n); fixed_lit(w, s); w.put(v, nb); w.code(0, 5)
        data += b"x" * n
    fixed_lit(w, 256)
    add("distance-1-every-length", w, bytes(data), "OK")
    return out


def mutations(streams):
    """(name, bytes, the status when it is certain or None) of byte flips and truncations at every offset of `streams`, a wrong
    CRC or ISIZE, zero padding, a second member and trailing garbage"""
    out = []
    for name, b in streams:
        for i in range(len(b)):
            for x in (0x01, 0x80, 0xFF):
                m = bytearray(b); m[i] ^= x
                out.append((f"{name}-flip{i}-{x}", bytes(m), None))
            out.append((f"{name}-cut{i}", b[:i], None))
        crc = bytearray(b); crc[-8] ^= 1
        out.append((f"{name}-crc", bytes(crc), "CRC"))
        size = bytearray(b); size[-4] ^= 1
        out.append((f"{name}-isize", bytes(size), "SIZE"))
        out.append((f"{name}-zero-padding", b + bytes(8), None))
        out.append((f"{name}-second-member", b + b, None))
        out.append((f"{name}-garbage", b + b"garbage!", None))
    return out


def slots(blobs):
    """the readers' slot rule: (index of every blob the device is given, its slot size); the rest go to the host"""
    take, size = [], []
    for i, b in enumerate(blobs):
        n = _logio.gz_isize(b)
        if n is not None:
            take.append(i); size.append(n)
    return take, size


def _pack(blobs):
    take, size = slots(blobs)
    gz = b"".join(blobs[i] for i in take)
    gz_off = np.zeros(len(take) + 1, dtype=np.int64); np.cumsum([len(blobs[i]) for i in take], out=gz_off[1:])
    out_off = np.zeros(len(take) + 1, dtype=np.int64); np.cumsum(size, out=out_off[1:])
    return take, np.frombuffer(gz, dtype=np.uint8).copy() if gz else np.zeros(8, dtype=np.uint8), gz_off, out_off


def emul_gunzip(blobs, sanitize=False):
    """per blob: None (left to the host) or (status name, output bytes) from the host emulation"""
    import emul_lib

    take, gz, gz_off, out_off = _pack(blobs)
    res = [None] * len(blobs)
    if not take:
        return res
    out = np.zeros(max(int(out_off[-1]), 1), dtype=np.uint8)
    st = np.zeros(len(take), dtype=np.int32)
    L = emul_lib.lib(sanitize=sanitize)
    assert L.emulz_gunzip(len(take), gz.ctypes.data, int(gz_off[-1]), gz_off.ctypes.data, out.ctypes.data, int(out_off[-1]),
                          out_off.ctypes.data, st.ctypes.data) == 0
    for j, i in enumerate(take):
        res[i] = (_logio.GUNZIP_STATUSES[st[j]].upper(), out[out_off[j]:out_off[j + 1]].tobytes())
    return res


def dev_gunzip(blobs, device=0):
    """the same through mjx_gunzip_dev on `device`, one launch for all blobs"""
    import torch

    from mortal_b200 import _lib

    _lib.init(device)
    take, gz, gz_off, out_off = _pack(blobs)
    res = [None] * len(blobs)
    if not take:
        return res
    dev = torch.device("cuda", device)
    d_gz = torch.from_numpy(gz).to(dev)
    d_go, d_oo = torch.from_numpy(gz_off).to(dev), torch.from_numpy(out_off).to(dev)
    out = torch.empty(max(int(out_off[-1]), 1), dtype=torch.uint8, device=dev)
    st = torch.full((len(take),), -1, dtype=torch.int32, device=dev)
    _lib.check(_logio._load().mjx_gunzip_dev(len(take), d_gz.data_ptr(), int(gz_off[-1]), d_go.data_ptr(), out.data_ptr(),
                                             int(out_off[-1]), d_oo.data_ptr(), st.data_ptr(), torch.cuda.current_stream(dev).cuda_stream),
               "mjx_gunzip_dev")
    o, s = out.cpu().numpy(), st.cpu().numpy()
    for j, i in enumerate(take):
        res[i] = (_logio.GUNZIP_STATUSES[s[j]].upper(), o[out_off[j]:out_off[j + 1]].tobytes())
    return res


def python_gunzip(b):
    """gzip.decompress(b), or None when it raises"""
    try:
        return gzip.decompress(b)
    except Exception:  # noqa: BLE001
        return None


def check_contract(name, b, got, want_status=None):
    """OK => the bytes gzip.decompress returns; gzip.decompress raising => not OK; and the expected status when one is given"""
    py = python_gunzip(b)
    if got is None:  # left to the host
        assert want_status is None or want_status != "OK", name
        return
    status, data = got
    if status == "OK":
        assert py is not None and py == data, name
    if py is None:
        assert status != "OK", name
    if want_status is not None:
        assert status == want_status, (name, status, want_status)
