"""k_mjai_decode on the GPU: arena logs (with `meta`) and format variations are all accepted and decode to the host path's arrays;
validate_logs gives the host-only path's verdicts on mixed corpora in any order and batching; the CLI prints what the host-only
path prints."""
import gzip
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import log_mutations as LM
import mjai_lib as M

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Eng:
    engine_type, version, is_oracle, enable_quick_eval, enable_rule_based_agari_guard, name = "mortal", 4, False, True, False, "e"

    def react_device(self, obs, masks):
        q = torch.rand(masks.shape, device=masks.device)
        q[:, :34] += 2.0 * obs[:, 876, :] + obs[:, 875, :]
        q = q.masked_fill(~masks, -1.0)
        return q.argmax(-1), q


@pytest.fixture(scope="module")
def arena_texts(tmp_path_factory):
    from mortal_b200.libriichi.arena import OneVsThree

    d = tmp_path_factory.mktemp("arena")
    OneVsThree(disable_progress_bar=True, log_dir=str(d)).py_vs_py(_Eng(), _Eng(), (78000, 13), 256)
    return [gzip.open(os.path.join(d, f), "rt").read() for f in sorted(os.listdir(d))]


def _device_arrays(texts, augment=False):
    """per log: None (declined) or the emul_decode-style dict, from decode_dev"""
    from mortal_b200.validate_logs import decode_dev

    blobs = [t.encode("utf-8") for t in texts]
    D = decode_dev(blobs, 0, augment)
    hdr, lines = D.hdr.cpu().numpy().view(np.uint64), D.lines.cpu().numpy()
    ky, ho = D.kyoku.cpu().numpy().view(np.uint64).reshape(-1, 19), D.hora.cpu().numpy().view(np.uint64).reshape(-1, 2)
    out = []
    for i, b in enumerate(blobs):
        a, e, k, h, fb, fe = (int(x) for x in D.counts[i])
        if not a:
            out.append(None)
            continue
        eo, ko, hoff = int(D.ev_off[i]), int(D.ky_off[i]), int(D.hora_off[i])
        out.append(dict(hdr=hdr[eo:eo + e], lines=lines[eo:eo + e], kyoku=ky[ko:ko + k], hora=ho[hoff:hoff + h], first=b[fb:fe]))
    return out


def test_arena_logs_decode_as_on_the_host(arena_texts):
    assert len(arena_texts) == 1024 and all('"meta"' in t for t in arena_texts[:8])
    got = _device_arrays(arena_texts)
    assert all(g is not None for g in got), sum(g is None for g in got)
    for t, g in zip(arena_texts, got):
        assert M.same(g, M.host_decode(t.encode("utf-8")))


def test_augment_on_the_device(arena_texts):
    got = _device_arrays(arena_texts[:64], augment=True)
    for t, g in zip(arena_texts[:64], got):
        assert g is not None and M.same(g, M.host_decode(t.encode("utf-8"), augment=True))


@pytest.fixture(scope="module")
def variations(arena_texts):
    rng = np.random.default_rng(41)
    games = [[json.loads(x) for x in t.splitlines()] for t in arena_texts[:128]]
    return [M.vary(g, rng) for g in games]


def test_format_variations_are_accepted(variations):
    got = _device_arrays(variations)
    assert all(g is not None for g in got), sum(g is None for g in got)
    for t, g in zip(variations, got):
        assert M.same(g, M.host_decode(t.encode("utf-8")))


def test_declines_before_long_newline_runs_leave_block_mates_intact(arena_texts):
    # every CTA of k_mjai_decode holds 4 logs: one declining log with a run of line breaks longer than the warp's 64-entry queue
    # of line ends, next to three logs that must decode exactly as on the host
    texts = []
    for k in range(64):
        bad = ("x" if k % 2 else '{"type":"start_game"}\nnot json') + "\n" * (128 + 37 * k)
        slot = k % 4
        group = list(arena_texts[3 * k:3 * k + 3])
        group.insert(slot, bad)
        texts += group
    got = _device_arrays(texts)
    for t, g in zip(texts, got):
        want = M.host_decode(t.encode("utf-8"))
        if want is None:
            assert g is None
        else:
            assert g is not None and M.same(g, want)
    assert sum(g is None for g in got) == 64


def _host_only(texts):
    """the verdicts of the host decoder + k_validate_logs (encode_log + run_packed)"""
    from mortal_b200.validate_logs import EncodedLog, Verdict, encode_log, pack, run_packed, to_verdict

    enc = [t if isinstance(t, Verdict) else encode_log(t) for t in texts]
    dev = [e for e in enc if isinstance(e, EncodedLog)]
    rows = run_packed(pack(dev)) if dev else None
    out, k = [], 0
    for e in enc:
        if isinstance(e, Verdict):
            out.append(e)
        else:
            out.append(to_verdict(rows[k], e)); k += 1
    return out, enc


@pytest.fixture(scope="module")
def mixed(arena_texts, variations):
    rng = np.random.default_rng(43)
    games = [[json.loads(x) for x in t.splitlines()] for t in arena_texts[:128]]
    mutated = [t for _, t in LM.mutated_corpus(games, 40, rng)]
    mutated += [M.vary([json.loads(x) for x in t.splitlines()], rng) for t in mutated[::7] if all(
        _parses(x) for x in t.splitlines() if x.strip())]
    hostile = []
    for _, b in M.hostile_corpus(arena_texts[:32] + variations[:32], 60, rng):
        try:
            hostile.append(b.decode("utf-8"))
        except UnicodeDecodeError:
            pass
    texts = variations + mutated + hostile + ["", "\n\n", "{}\n", "\ud800"]
    return texts, _host_only(texts)[0]


def _parses(x):
    try:
        json.loads(x)
        return True
    except ValueError:
        return False


def test_mixed_corpora_get_the_host_verdicts(mixed):
    from mortal_b200.validate_logs import validate_logs

    texts, want = mixed
    assert len(texts) > 1000
    assert validate_logs(texts) == want
    perm = np.random.default_rng(5).permutation(len(texts))
    shuffled = validate_logs([texts[i] for i in perm])
    assert [shuffled[int(np.where(perm == i)[0][0])] for i in range(len(texts))] == want
    parts = []
    for lo, hi in ((0, 1), (1, 300), (300, 301), (301, len(texts))):
        parts += validate_logs(texts[lo:hi])
    assert parts == want


def test_cli_prints_what_the_host_path_prints(arena_texts, tmp_path):
    from mortal_b200.validate_logs import _read, message

    events = [json.loads(x) for x in arena_texts[0].splitlines()]
    bad = next(t for s in range(50) for t in [LM.mutate(events, "riichi_not_tenpai", np.random.default_rng(s))] if t is not None)
    layout = {"a/ok1.json": arena_texts[1], "a/b/ok2.json.gz": arena_texts[2], "bad.json.gz": bad,
              "crlf.json": arena_texts[3].replace("\n", "\r\n"), "crlf_bad.json.gz": bad.replace("\n", "\r\n"),
              "a/bad2.json": "{\"type\": \"start_game\"}\nnot json\n"}
    for name, text in layout.items():
        p = tmp_path / name
        p.parent.mkdir(parents=True, exist_ok=True)
        if name.endswith(".gz"):
            with gzip.open(p, "wt", newline="") as f:
                f.write(text)
        else:
            p.write_bytes(text.encode("utf-8"))
    (tmp_path / "latin1.json").write_bytes(b'{"type":"start_game","names":["caf\xe9"]}\n')
    (tmp_path / "notgz.json.gz").write_bytes(b"plain text, not gzip")
    paths = sorted(str(p) for p in tmp_path.rglob("*") if p.name.endswith((".json", ".json.gz")))
    verdicts, enc = _host_only([_read(p) for p in paths])
    want = "".join(f"\nerror in log {p}\n{message(v, e)}\n" for p, v, e in zip(paths, verdicts, enc) if v is not None)
    r = subprocess.run([sys.executable, "-m", "mortal_b200.validate_logs", str(tmp_path)], cwd=ROOT, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr
    assert r.stdout == want
    assert r.stdout.count("error in log ") == 5
