"""Helpers of the mjai decoder tests — TEST INFRASTRUCTURE: the host build of csrc/mjx_mjai.cuh (tests/host_emul/emul_mjai.cc),
the host path's arrays for comparison, and two seeded corpora: format variations Python's json reads exactly as the canonical
text, and byte-level hostile mutations."""
from __future__ import annotations

import ctypes as C
import json
import os

import numpy as np

import emul_lib as E
from mortal_b200 import dataset_codec
from mortal_b200.validate_logs import EncodedLog, encode_log

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def emul_lib():
    """emul_lib.lib() with the emulated decoder's entry declared"""
    L = E.lib()
    L.emulm_decode.argtypes = [C.c_int, C.c_void_p, C.c_longlong, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong]
    return L


def emul_decode(blobs, augment=False):
    """bytes per log -> per log None (declined) or dict(hdr, kyoku [k, 19], hora [h, 2], lines, first = bytes of the first event
    line), through the count and fill calls of the emulated decoder"""
    L = emul_lib()
    n = len(blobs)
    buf = np.frombuffer(b"".join(blobs) or b"\0", dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(b) for b in blobs], out=off[1:])
    counts = np.zeros((n, 6), dtype=np.int32)
    nb = int(off[-1])
    assert L.emulm_decode(n, buf.ctypes.data, nb, off.ctypes.data, int(augment), counts.ctypes.data, None, None, None, None, None, 0,
                          None, 0, None, 0) == 0
    excl = lambda x: (np.cumsum(x) - x).astype(np.int32)
    eo, ko, ho = excl(counts[:, 1]), excl(counts[:, 2]), excl(counts[:, 3])
    ne, nk, nh = (int(counts[:, k].sum()) for k in (1, 2, 3))
    hdr, lines = np.zeros(max(ne, 1), dtype=np.uint64), np.zeros(max(ne, 1), dtype=np.int32)
    ky, hora = np.zeros(max(nk, 1) * 19, dtype=np.uint64), np.zeros(max(nh, 1) * 2, dtype=np.uint64)
    assert L.emulm_decode(n, buf.ctypes.data, nb, off.ctypes.data, int(augment), counts.ctypes.data, eo.ctypes.data, ko.ctypes.data,
                          ho.ctypes.data, hdr.ctypes.data, lines.ctypes.data, ne, ky.ctypes.data, nk * 19, hora.ctypes.data, nh * 2) == 0
    out = []
    for i in range(n):
        a, e, k, h, fb, fe = (int(x) for x in counts[i])
        if not a:
            out.append(None)
            continue
        out.append(dict(hdr=hdr[eo[i]:eo[i] + e], kyoku=ky[ko[i] * 19:(ko[i] + k) * 19].reshape(-1, 19),
                        hora=hora[ho[i] * 2:(ho[i] + h) * 2].reshape(-1, 2), lines=lines[eo[i]:eo[i] + e], first=blobs[i][fb:fe]))
    return out


def host_decode(blob: bytes, augment=False):
    """what the host path makes of a log's bytes: the dict emul_decode returns, or None where the host rejects or special-cases
    the log (not UTF-8, a parse or structural error, no events)"""
    try:
        text = blob.decode("utf-8")
        e = encode_log(text)
    except Exception:  # noqa: BLE001 — any failure on the host must be a decline on the device
        return None
    if not isinstance(e, EncodedLog) or not e.lines:
        return None
    hdr, ky, hora = e.hdr, e.kyoku, e.hora
    if augment:
        hl = []
        hdr, ky = dataset_codec.encode_events(dataset_codec.augment_events([json.loads(t) for t in e.texts]), hora=hl)
        hora = np.array(hl, dtype=np.uint64).reshape(-1, 2)
    return dict(hdr=hdr, kyoku=ky, hora=hora, lines=np.array(e.lines, dtype=np.int32), first=e.texts[0].encode("utf-8"))


def same(a, b) -> bool:
    return all(np.array_equal(np.asarray(a[k], dtype=np.int64), np.asarray(b[k], dtype=np.int64)) for k in ("hdr", "kyoku", "hora", "lines")) \
        and a["first"] == b["first"]


def golden_texts():
    """the mjai logs under tests/golden: the reference's golden game and the state tests' logs"""
    out = [open(os.path.join(ROOT, "tests", "golden", "golden_game.jsonl"), encoding="utf-8").read()]
    with open(os.path.join(ROOT, "tests", "golden", "state_test_logs.json"), encoding="utf-8") as f:
        for logs in json.load(f).values():
            for lg in logs:
                out.append("\n".join(x if isinstance(x, str) else json.dumps(x) for x in lg) + "\n")
    return out


def game_text(events) -> str:
    return "\n".join(json.dumps(e, separators=(",", ":"), ensure_ascii=False) for e in events) + "\n"


# ---- format variations: every one is read by Python's json exactly as the canonical line ----------------------------------------
_EXTRA = ['-0', '0', '1.5e-3', '1E+2', '-12.25E7', '123456789012345678901234567890', '0.0', '-1e-0', 'true', 'false', 'null', '""',
          '[]', '{}', '[1, -2.0, {"a": [true, false, null]}]', '{"k\\u00e9y": "v\\n\\"\\\\\\/\\b\\f\\r\\t\\u2028", "deep": [[[[{}]]]]}',
          '"\\ud83d\\ude00 \\u00fc"', '{"q_values":[0.125,-2.5e-05,3],"mask_bits":70368744177663,"is_greedy":true,'
          '"kan_select":{"q_values":[1.0],"mask_bits":4398046511104}}', '"café 名"', '[[[[[[[[[[[[[[[[1]]]]]]]]]]]]]]]]']


def _ws(rng):
    return ["", " ", "\t", "  ", " \t "][int(rng.integers(5))]


def _dump_var(o, rng, ensure_ascii, top=False):
    if isinstance(o, dict):
        items = list(o.items())
        rng.shuffle(items)
        parts = [json.dumps(k, ensure_ascii=ensure_ascii) + _ws(rng) + ":" + _ws(rng) + _dump_var(v, rng, ensure_ascii) for k, v in items]
        if top and rng.integers(2):
            for _ in range(int(rng.integers(1, 4))):
                parts.insert(int(rng.integers(len(parts) + 1)), f'"x{int(rng.integers(100))}_extra"' + _ws(rng) + ":" + _ws(rng)
                             + _EXTRA[int(rng.integers(len(_EXTRA)))])
        return "{" + _ws(rng) + ("," + _ws(rng)).join(parts) + _ws(rng) + "}"
    if isinstance(o, list):
        return "[" + _ws(rng) + ("," + _ws(rng)).join(_dump_var(v, rng, ensure_ascii) for v in o) + _ws(rng) + "]"
    return json.dumps(o, ensure_ascii=ensure_ascii)


def vary(events, rng) -> str:
    """one log in a random format: shuffled keys, spaces and tabs between tokens, "\\n" or "\\r\\n", blank lines, ensure_ascii
    on or off, unknown fields of every JSON form; names with non-ASCII letters"""
    ev = [dict(e) for e in events]
    if ev and ev[0].get("type") == "start_game":
        ev[0]["names"] = ["Ｍortal", "café", "名前", "a\"b\\c"]
    ensure_ascii = bool(rng.integers(2))
    nl = "\r\n" if rng.integers(2) else "\n"
    lines = []
    for e in ev:
        if rng.integers(8) == 0:
            lines.append(["", " ", "\t", " \t "][int(rng.integers(4))])
        lines.append(_ws(rng) + _dump_var(e, rng, ensure_ascii, top=True) + _ws(rng))
    return nl.join(lines) + (nl if rng.integers(4) else "")


# ---- hostile mutations: bytes the device must decline, or decode exactly as the host ------------------------------------------
HOSTILE = ("insert", "delete", "replace", "truncate", "dup_key", "nan", "float_actor", "key_escape", "u2028", "lone_cr", "control",
           "non_object", "trailing", "deep", "bad_utf8", "newline_run")


def hostile(text: str, cls: str, rng) -> bytes:
    b = bytearray(text.encode("utf-8"))
    lines = text.split("\n")
    pick = lambda: int(rng.integers(len(lines)))

    def edit_line(f):
        cands = [i for i, ln in enumerate(lines) if ln.strip()]
        i = cands[int(rng.integers(len(cands)))]
        lines[i] = f(lines[i])
        return "\n".join(lines).encode("utf-8")

    def sub_actor(ln, rep):
        k = ln.find('"actor":')
        return ln if k < 0 else ln[:k + 8] + rep + ln[k + 9:]

    if cls == "insert":
        b.insert(int(rng.integers(len(b) + 1)), int(rng.integers(0, 128)))
    elif cls == "delete":
        del b[int(rng.integers(len(b)))]
    elif cls == "replace":
        b[int(rng.integers(len(b)))] = int(rng.integers(0, 128))
    elif cls == "truncate":
        b = b[:int(rng.integers(len(b)))]
    elif cls == "dup_key":
        return edit_line(lambda ln: ln.replace('"type":', '"type":"dahai","type":', 1) if rng.integers(2) else
                         ln.replace("{", '{"pai":"1m",', 1).replace('"pai":"1m",', '"pai":"1m","pai":"2m",', 1))
    elif cls == "nan":
        return edit_line(lambda ln: ln.replace("{", '{"x":' + ["NaN", "Infinity", "-Infinity"][int(rng.integers(3))] + ",", 1))
    elif cls == "float_actor":
        return edit_line(lambda ln: sub_actor(ln, ["1.0", "1e0", "true", "-1", "4", "01"][int(rng.integers(6))]))
    elif cls == "key_escape":
        return edit_line(lambda ln: ln.replace('"type"', '"typ\\u0065"', 1) if rng.integers(2) else ln.replace('"actor"', '"\\u0061ctor"', 1))
    elif cls == "u2028":
        return edit_line(lambda ln: ln.replace("{", '{"names":["a\u2028b"],', 1) if rng.integers(2) else
                         ln.replace("{", '{"n":"\u0085 ",', 1))
    elif cls == "lone_cr":
        b.insert(int(rng.integers(len(b) + 1)), 13)
    elif cls == "control":
        return edit_line(lambda ln: ln.replace("{", '{"x":"a' + chr(int(rng.choice([0, 9, 10, 11, 12, 27, 28, 31]))) + 'b",', 1))
    elif cls == "non_object":
        lines.insert(pick(), ["[1,2]", '"start_game"', "3", "null", "{", "}", "{}"][int(rng.integers(7))])
        return "\n".join(lines).encode("utf-8")
    elif cls == "trailing":
        return edit_line(lambda ln: ln.rstrip() + ["x", " {}", ",", "}", " 1"][int(rng.integers(5))])
    elif cls == "deep":
        d = int(rng.integers(33, 40))  # deeper than MJAI_DEPTH
        return edit_line(lambda ln: ln.replace("{", '{"x":' + "[" * d + "]" * d + ",", 1))
    elif cls == "bad_utf8":
        b[int(rng.integers(len(b)))] = int(rng.choice([0x80, 0xC0, 0xFF, 0xE2]))
    elif cls == "newline_run":  # a line Python rejects, then more line breaks than the decoder queues at once
        lines.insert(pick(), "not json" + "\n" * int(rng.integers(100, 400)))
        return "\n".join(lines).encode("utf-8")
    else:
        raise ValueError(cls)
    return bytes(b)


def hostile_corpus(texts, n_per_class, rng):
    """[(class, bytes)]: n_per_class mutations of every class, each of a randomly chosen text"""
    return [(c, hostile(texts[int(rng.integers(len(texts)))], c, rng)) for c in HOSTILE for _ in range(n_per_class)]
