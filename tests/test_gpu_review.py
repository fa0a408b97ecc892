"""mortal_b200.review on the GPU: the batched review equals libriichi.mjai.Bot on the CUDA PlayerState, driven line by line as
mortal.py's review mode drives it, byte for byte with meta.eval_time_ns masked."""
import gzip
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_game.jsonl")


def _dumps(events):
    return "".join(json.dumps(e, separators=(",", ":")) + "\n" for e in events)


@pytest.fixture(scope="module")
def cuda_state():
    from mortal_b200.libriichi import state

    prev = state._backend
    state.set_backend(state._CudaBackend())
    yield
    state.set_backend(prev)


@pytest.fixture(scope="module")
def logs():
    """(text, seats): the golden game, emulated self-play games of both test-policy kinds, and single-viewpoint versions"""
    import review_lib
    import validate_lib
    import viewpoint_lib

    out = [(open(GOLDEN).read(), [0, 1, 2, 3])]
    for policy in (0, 1):
        games = validate_lib.emul_games(2, policy, seed0=771000 + 100 * policy)
        out += [(_dumps(g), [0, 1, 2, 3]) for g in games]
        out += [(_dumps(viewpoint_lib.viewpoint(g, p)), [p]) for p, g in zip((1, 2), games)]
        out += [(_dumps(ev), ps) for ev, ps in review_lib.guard_logs(validate_lib.emul_games(4, policy, seed0=772000 + 100 * policy))]
    return out


def _check_parity(engine, logs, inputs):
    import review_lib

    from mortal_b200.review import review_logs

    got = review_logs(engine, inputs, [s for _, s in logs])
    for (text, seats), rs in zip(logs, got):
        assert [r.player_id for r in rs] == seats
        for r in rs:
            assert r.error is None, r.error
            want = review_lib.bot_review(engine, text, r.player_id)
            assert review_lib.mask_eval(r.text) == review_lib.mask_eval(want)
    return got


@pytest.mark.parametrize("guard", [True, False])
def test_stub_review_equals_the_bot(cuda_state, logs, guard):
    import review_lib

    engine = review_lib.DeviceStubEngine(guard)
    got = _check_parity(engine, logs, [t for t, _ in logs])
    # what the run exercised
    text = "".join(r.text for rs in got for r in rs)
    for kind in ("dahai", "chi", "pon", "reach", "hora"):
        assert f'{{"type":"{kind}"' in text, kind
    assert '{"type":"none","meta":{"q_values"' in text  # a pass
    assert review_lib.NONE_LINE in text
    lines = text.splitlines()
    assert any(ln.startswith('{"type":"ankan"') and '"kan_select":{' in ln for ln in lines)
    assert any(ln.startswith('{"type":"kakan"') and '"kan_select":{' in ln for ln in lines)
    labels = np.concatenate([r.label.cpu().numpy() for rs in got for r in rs])
    assert (labels >= 0).any() and (labels < 0).any()
    # the agari guard is the only reason a reaction differs from the engine's argmax
    for rs in got:
        for r in rs:
            differs = r.q_values.argmax(-1) != r.action
            assert guard or not differs.any()
            assert (r.q_values.argmax(-1)[differs] == 43).all()
    over = sum(int((r.q_values.argmax(-1) != r.action).sum()) for rs in got for r in rs)
    assert (over > 0) == guard
    for rs in got:  # one line per event
        for r in rs:
            assert r.event_index.numel() == r.action.numel() == r.q_values.shape[0] == r.masks.shape[0]


def test_gz_paths_and_host_engine(cuda_state, logs, tmp_path):
    """.json.gz and .json files (gunzipped on the device when there are enough of them), and a react_batch-only engine"""
    import review_lib

    from mortal_b200 import _logio

    reps = -(-2 * _logio.GZ_DEVICE_MIN_FILES // len(logs))  # enough .json.gz files for the device gunzip
    many = logs * reps
    paths = []
    for i, (text, _) in enumerate(many):
        p = tmp_path / (f"{i}.json.gz" if i % 2 == 0 else f"{i}.json")
        if i % 2 == 0:
            with gzip.open(p, "wt") as f:
                f.write(text)
        else:
            p.write_text(text)
        paths.append(str(p))
    assert sum(p.endswith(".gz") for p in paths) >= _logio.GZ_DEVICE_MIN_FILES
    from mortal_b200.review import review_logs

    engine = review_lib.DeviceStubEngine(True)
    want = {t: [review_lib.mask_eval(review_lib.bot_review(engine, t, p)) for p in seats] for t, seats in logs}
    got = review_logs(engine, paths, [s for _, s in many])
    for (text, _), rs in zip(many, got):
        assert [review_lib.mask_eval(r.text) for r in rs] == want[text]
    host = review_lib.StubEngine(True)
    got = _check_parity(host, logs[:2], [t for t, _ in logs[:2]])
    assert got[0][0].text.count("\n") == sum(1 for ln in logs[0][0].splitlines() if ln.strip())


def test_fallbacks_and_errors(cuda_state, logs):
    """logs with can_act go through the Bot; a mutated log is reviewed as the Bot reviews it; a reaction that cannot be decoded fails
    its job alone at the Bot's event; a log hiding the seat's own tiles fails that seat alone with error code 13"""
    import review_lib

    from mortal_b200.review import review_logs

    engine = review_lib.DeviceStubEngine(True)
    text = logs[1][0]
    lines = text.splitlines()
    with_can_act = "\n".join(ln[:-1] + ',"can_act":true}' if '"tsumo"' in ln else ln for ln in lines) + "\n"
    bad = lines[:]
    k = next(i for i, ln in enumerate(bad) if '"dahai"' in ln and i > 20)
    ev = json.loads(bad[k])
    actor = ev["actor"]
    from mortal_b200.libriichi.state import PlayerState
    from mortal_b200.mjai_log import TILE_NAMES

    tehai = PlayerState.from_log(actor, bad[:k]).tehai
    ev["pai"] = TILE_NAMES[next(t for t in range(27, 34) if tehai[t] == 0)]  # an honour the actor does not hold
    ev["tsumogiri"] = False
    bad[k] = json.dumps(ev, separators=(",", ":"))
    bad_text = "\n".join(bad) + "\n"
    hidden = logs[3]  # a viewpoint log of one seat
    own = hidden[1][0]
    got = review_logs(engine, [with_can_act, bad_text, hidden[0], text], [[0], [0, 1, 2, 3], [(own + 1) % 4, own], [2]])
    assert got[0][0].error is None
    assert review_lib.mask_eval(got[0][0].text) == review_lib.mask_eval(review_lib.bot_review(engine, with_can_act, 0))
    for r in got[1]:  # the state follows the mutated log as the Bot's does
        assert r.error is None
        assert review_lib.mask_eval(r.text) == review_lib.mask_eval(review_lib.bot_review(engine, bad_text, r.player_id))
    illegal = review_lib.DeviceIllegalStubEngine(True)  # reactions that cannot be decoded: the job fails at the Bot's event
    got_i = review_logs(illegal, [text], [[0, 1, 2, 3]])[0]
    failed = 0
    for r in got_i:
        at = review_lib.bot_fail_index(illegal, text, r.player_id)
        if at is None:
            assert r.error is None and review_lib.mask_eval(r.text) == review_lib.mask_eval(review_lib.bot_review(illegal, text, r.player_id))
        else:
            assert r.text is None and f"at event {at} with mjx error code 1" in r.error, r.error
            failed += 1
    assert failed > 0
    assert got[2][0].text is None and "code 13" in got[2][0].error
    assert got[2][1].error is None
    assert got[3][0].error is None


def test_rejections():
    import review_lib

    from mortal_b200.review import review_logs

    quick = review_lib.DeviceStubEngine(True)
    quick.enable_quick_eval = True
    oracle = review_lib.DeviceStubEngine(True)
    oracle.is_oracle = True
    for e in (quick, oracle):
        with pytest.raises(ValueError):
            review_logs(e, ["{}"], [0])


def _lines(text):
    return [json.loads(ln) for ln in text.splitlines()]


@pytest.mark.parametrize("version", [2, 3, 4])
@pytest.mark.parametrize("fast", [False, True])
def test_checkpoints(cuda_state, logs, version, fast):
    """real checkpoints against the per-line Bot with the same engine. fp32 (TF32 off): the two differ only in summation order
    (batch size picks other cuDNN / cuBLAS kernels), a few ulp of values of order 1-10, so 1e-3 absolute. bf16 DeviceEngine: the
    activations are rounded to 8-bit mantissas at every layer whatever the batch, and a different reduction order moves a Q-value
    by a few bf16 ulp of the pre-head activations; 0.1 absolute covers that with margin. Reactions must agree wherever the
    legal top-two gap exceeds twice the tolerance."""
    import torch

    import mortal_ckpt
    from mortal_b200.engine import DeviceEngine
    from mortal_b200.model import load_mortal
    from mortal_b200.review import review_logs

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    fx = mortal_ckpt.load_fixture()
    brain, dqn = load_mortal(mortal_ckpt.checkpoint(f"v{version}", fx[f"v{version}"]))
    engine = DeviceEngine(brain, dqn, version=version, enable_amp=fast, enable_quick_eval=False, enable_rule_based_agari_guard=True)
    tol = 0.1 if fast else 1e-3
    sel = logs[:2]
    got = review_logs(engine, [t for t, _ in sel], [s for _, s in sel])
    for (text, _), rs in zip(sel, got):
        for r in rs:
            assert r.error is None, r.error
            a, b = _lines(r.text), _lines(review_lib_bot(engine, text, r.player_id))
            assert len(a) == len(b)
            for x, y in zip(a, b):
                if "q_values" not in y["meta"]:
                    assert x == y
                    continue
                for m, n in ((x["meta"], y["meta"]),) + (((x["meta"]["kan_select"], y["meta"]["kan_select"]),)
                                                          if "kan_select" in x["meta"] and "kan_select" in y["meta"] else ()):
                    for key in ("mask_bits", "shanten", "at_furiten", "batch_size", "is_greedy"):
                        assert m[key] == n[key], key
                    np.testing.assert_allclose(m["q_values"], n["q_values"], atol=tol, rtol=0)
                q = sorted(y["meta"]["q_values"], reverse=True)
                if len(q) < 2 or q[0] - q[1] > 2 * tol:
                    assert {k: v for k, v in x.items() if k != "meta"} == {k: v for k, v in y.items() if k != "meta"}


def review_lib_bot(engine, text, seat):
    import review_lib

    return review_lib.bot_review(engine, text, seat)


def test_phi_matrix_and_clis(cuda_state, logs, tmp_path):
    """the extra_data line against reward_lib's float64 restatement; the mortal and review command lines in subprocesses"""
    import copy
    import subprocess
    import sys

    import torch

    import mortal_ckpt
    import reward_lib
    from mortal_b200.dataset import Grp
    from mortal_b200.mortal import load_engine, load_review_engine
    from mortal_b200.review import review_logs

    fx = mortal_ckpt.load_fixture()
    ckpt = mortal_ckpt.checkpoint("v4", fx["v4"])
    ckpt["tag"] = "test-tag"
    grp = reward_lib.random_grp(64, 2, 5)
    torch.save(ckpt, tmp_path / "mortal.pth")
    torch.save({"model": grp.state_dict()}, tmp_path / "grp.pth")
    cfg = tmp_path / "config.toml"
    cfg.write_text(f'[control]\nstate_file = "{tmp_path / "mortal.pth"}"\n[grp]\nstate_file = "{tmp_path / "grp.pth"}"\n'
                   "[grp.network]\nhidden_size = 64\nnum_layers = 2\n")
    config = {"control": {"state_file": str(tmp_path / "mortal.pth")}, "grp": {"state_file": str(tmp_path / "grp.pth")}}
    engine, grp_state, tag = load_review_engine(config)
    assert tag == "test-tag"
    text = logs[0][0]
    (r,), = review_logs(engine, [text], [1], grp=grp_state, model_tag=tag)
    extra = json.loads(r.text.splitlines()[-1])
    assert extra["model_tag"] == "test-tag"
    ref = reward_lib.ref_calc_grp(copy.deepcopy(grp).double(), Grp.load_log(text).take_feature())
    np.testing.assert_allclose(np.array(extra["phi_matrix"]), ref.numpy(), rtol=0, atol=1e-12)

    env = dict(os.environ, MORTAL_CFG=str(cfg), PYTHONPATH=ROOT)
    run = lambda args, inp, **kw: subprocess.run([sys.executable, "-m", *args], input=inp, capture_output=True, text=True, cwd=ROOT,
                                                 env=dict(env, **kw), timeout=900)
    out = run(["mortal_b200.mortal", "1"], text, MORTAL_REVIEW_MODE="1")
    assert out.returncode == 0, out.stderr
    n_in = sum(1 for ln in text.splitlines() if ln.strip())
    assert len(out.stdout.splitlines()) == n_in + 1
    import review_lib

    assert review_lib.mask_eval(out.stdout) == review_lib.mask_eval(r.text)
    live = run(["mortal_b200.mortal", "1"], text)
    assert live.returncode == 0, live.stderr
    le, _ = load_engine(False, config)
    want = [ln.strip() for ln in text.splitlines() if ln.strip()]
    from mortal_b200.libriichi.mjai import Bot

    bot = Bot(le, 1)
    reacts = [x for x in (bot.react(ln) for ln in want) if x]
    assert review_lib.mask_eval(live.stdout) == review_lib.mask_eval("".join(x + "\n" for x in reacts))

    src, dst = tmp_path / "logs", tmp_path / "out"
    src.mkdir()
    name = json.loads(text.splitlines()[0])["names"][1]
    with gzip.open(src / "a.json.gz", "wt") as f:
        f.write(text)
    (src / "b.json").write_text(text)
    cli = run(["mortal_b200.review", str(src), name, str(dst)], "")
    assert cli.returncode == 0, cli.stderr
    summary = json.loads(cli.stdout.splitlines()[-1])
    seats = [s for s, nm in enumerate(json.loads(text.splitlines()[0])["names"]) if nm == name]
    both = review_logs(engine, [str(src / "a.json.gz"), str(src / "b.json")], [seats, seats], grp=grp_state, model_tag=tag)
    dec = lab = match = 0
    for stem, rs in zip(("a", "b"), both):
        for rv in rs:
            assert review_lib.mask_eval((dst / f"{stem}.{rv.player_id}.jsonl").read_text()) == review_lib.mask_eval(rv.text)
            dec += rv.action.numel(); lab += int((rv.label >= 0).sum()); match += int(((rv.action == rv.label) & (rv.label >= 0)).sum())
    assert summary == {"logs": 2, "decisions": dec, "labelled": lab, "matching": match, "failed": 0}
