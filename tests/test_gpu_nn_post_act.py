"""The version-1 and oracle-stem kernels of csrc/mjx_nn.cuh against the float64 references of nn_ref_post.py, at the shapes
and edges they run at; the version-1 and version-4-oracle networks layer by layer; every version end to end on arena rows."""
import ctypes as C
import math

import numpy as np
import pytest

import nn_ref as R
import nn_ref_post as P
from test_gpu_nn_numerics import (BATCHES, CHANNELS, LARGE, LENGTHS, ConvStats, _nan_like, _p, _sm, _special_floats, _stream, act,
                                  affine_params, b_gate, b_stream, gate_params, hidden_sizes)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import torch

    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from mortal_b200 import _lib

    _lib.init(0)
    return torch.device("cuda", 0)


def call_affine_relu(x, scale, bias):
    from mortal_b200 import _lib

    out = _nan_like(x)
    _lib.check(_lib.load().mjx_nn_affine_relu_bf16(_p(x), _p(scale), _p(bias), _p(out), x.numel(), x.shape[1], _stream()), "affine_relu")
    return out


def call_post_tail(y, x, scale, bias, w1, b1, w2t, b2):
    """(gate, x_out) through mjx_nn_post_block_tail_bf16 with buffers the test owns"""
    import torch

    from mortal_b200 import _lib

    b, c, _, l = y.shape
    gate = torch.full((b, c), float("nan"), dtype=torch.bfloat16, device=y.device)
    x_out = _nan_like(y)
    _lib.check(_lib.load().mjx_nn_post_block_tail_bf16(_p(y), _p(x), _p(scale), _p(bias), _p(w1), _p(b1), _p(w2t), _p(b2), _p(gate),
                                                       _p(x_out), b, l, c, w1.shape[0], _stream()), "post_block_tail")
    return gate, x_out


def check_affine_relu(x, scale, bias, got, what):
    v = P.affine_relu(x, scale, bias)
    R.check_within(f"{what} affine_relu", got, v, P.bound_affine_relu(v), R.NHWC_DIMS)


def check_post_tail(y, x, scale, bias, params, gate, x_out, what):
    b, c, _, l = y.shape
    g, zabs = P.post_gate(y, scale, bias, *params)
    R.check_within(f"{what} gate", gate, g, P.bound_post_gate(g, zabs, l, c, params[0].shape[0]), R.BC_DIMS)
    v, sa = P.post_residual(y, scale, bias, gate, x)
    R.check_within(f"{what} x_out", x_out, v, P.bound_post_residual(v, sa), R.NHWC_DIMS)
    return g


def test_affine_relu_every_shape_and_large_batches(dev):
    import torch

    gen = torch.Generator(device="cuda").manual_seed(21)
    for c in CHANNELS:
        scale, bias = affine_params(c, gen)
        for l in LENGTHS:
            for b in BATCHES:
                x = act(b, c, l, gen)
                check_affine_relu(x, scale, bias, call_affine_relu(x, scale, bias), f"B={b} C={c} L={l}")
    sm = _sm()
    for c, l in LARGE:
        b = b_stream(c, l, sm)
        scale, bias = affine_params(c, gen)
        x = act(b, c, l, gen)
        check_affine_relu(x, scale, bias, call_affine_relu(x, scale, bias), f"B={b} C={c} L={l}")
        del x
        torch.cuda.empty_cache()


def test_affine_relu_every_bf16_input(dev):
    """all 65536 bf16 patterns (±0, subnormals, ±inf, NaN, bf16-max) through 8 channel affines, negative scales among them and
    one that takes the pre-activation past the fp32 range"""
    import torch

    pat = torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).view(torch.bfloat16)
    scale = torch.tensor([1, -1, 2, -3.3, 1 + 2 ** -12, 1e-3, 0.5, -0.01], dtype=torch.float32, device="cuda")
    bias = torch.tensor([0, 0, 0, 0.1, 2 ** -9, -1e-38, 3e-39, -2.5], dtype=torch.float32, device="cuda")
    l = 32
    x = pat.view(-1, 1, 1, l).expand(-1, 8, 1, l).permute(0, 3, 2, 1).contiguous().permute(0, 3, 2, 1)
    got = call_affine_relu(x, scale, bias)
    check_affine_relu(x, scale, bias, got, "all bf16 inputs")
    t = R.pre_activation(x, scale, bias)
    g = got.double()
    assert torch.isnan(g[torch.isnan(t)]).all() and (g[t == -math.inf] == 0).all() and (g[t == math.inf] == math.inf).all()
    assert (g[torch.isfinite(t) & (t > 3.4e38)] == math.inf).all() and (g[t < 0] == 0).all()


def test_post_block_tail_every_shape(dev):
    """the gate against float64 of the post-affine pooling (negative BN scales; all-negative windows in some rows), x_out
    against float64 given the kernel's gate"""
    import torch

    gen = torch.Generator(device="cuda").manual_seed(22)
    spans = []
    for c in CHANNELS:
        scale, bias = affine_params(c, gen)
        for h in hidden_sizes(c):
            params = gate_params(c, h, gen)
            for l in LENGTHS:
                for b in BATCHES:
                    y, x = act(b, c, l, gen), act(b, c, l, gen)
                    if b == 7:
                        y[::2] = -y[::2].abs()  # every t of a negative-scale channel is then above its bias: max and min swap
                    what = f"B={b} C={c} H={h} L={l}"
                    gate, x_out = call_post_tail(y, x, scale, bias, *params)
                    g = check_post_tail(y, x, scale, bias, params, gate, x_out, what)
                    if b == 257:
                        spans.append((g.min().item(), g.max().item()))
    assert sum(lo < 0.1 and hi > 0.9 for lo, hi in spans) > len(spans) // 2, spans


def test_post_block_tail_pools_after_the_affine(dev):
    """all scales negative and every window of y positive: pooling y first and applying the affine after would take the max of
    t at the max of y, which is its minimum; the gate must match float64 of the post-affine pooling, and differ from the other"""
    import torch

    gen = torch.Generator(device="cuda").manual_seed(23)
    c, l, b = 64, 34, 33
    y = act(b, c, l, gen).abs() + 0.5
    x = act(b, c, l, gen)
    scale = -(torch.rand(c, generator=gen, device="cuda") + 0.5)
    bias = torch.randn(c, generator=gen, device="cuda")
    params = gate_params(c, 4, gen)
    gate, x_out = call_post_tail(y, x, scale, bias, *params)
    check_post_tail(y, x, scale, bias, params, gate, x_out, "negative scales")
    t = R.pre_activation(y, scale, bias).flatten(2)
    w1, b1, w2t, b2 = (R.f64(p) for p in params)
    wrong = 0
    for v in (t.mean(-1), R.f64(y).flatten(2).amax(-1) * R.f64(scale) + R.f64(bias)):
        wrong = wrong + torch.relu(v @ w1.T + b1) @ w2t + b2
    assert (torch.sigmoid(wrong) - gate.double()).abs().max() > 0.01


def test_post_block_tail_large_batches_and_edges(dev):
    """B_stream and B_gate rows (every grid-stride and row loop repeats); ±inf, NaN and subnormals in y and x; a NaN in one row
    stays in that row"""
    import torch

    gen = torch.Generator(device="cuda").manual_seed(24)
    sm = _sm()
    for c, l in LARGE:
        scale, bias = affine_params(c, gen)
        params = gate_params(c, c // 16, gen)
        for b in sorted({b_stream(c, l, sm), b_gate(sm)}):
            y, x = act(b, c, l, gen), act(b, c, l, gen)
            gate, x_out = call_post_tail(y, x, scale, bias, *params)
            check_post_tail(y, x, scale, bias, params, gate, x_out, f"B={b} C={c} L={l}")
            del y, x, gate, x_out
            torch.cuda.empty_cache()
    c, l, b = 64, 34, 9
    scale, bias = affine_params(c, gen)
    params = gate_params(c, 4, gen)
    y, x = act(b, c, l, gen), act(b, c, l, gen)
    x[1] = R.rn_bf16(torch.rand(c, 1, l, generator=gen, device="cuda").double() * 1e-38)  # subnormal residuals
    y[2] = R.rn_bf16(torch.rand(c, 1, l, generator=gen, device="cuda").double() * 1e-38)
    x[3, :, 0, 5] = math.inf
    x[4, :, 0, 6] = -math.inf
    clean = call_post_tail(y, x, scale, bias, *params)
    check_post_tail(y, x, scale, bias, params, *clean, "edges")
    assert (clean[1][3, :, 0, 5] == math.inf).all() and (clean[1][4, :, 0, 6] == 0).all()
    y[7, 11, 0, 3] = math.nan
    dirty = call_post_tail(y, x, scale, bias, *params)
    keep = torch.ones(b, dtype=torch.bool, device="cuda")
    keep[7] = False
    for d, cl in zip(dirty, clean):
        assert torch.isnan(d[7]).all() and torch.equal(d[keep].view(torch.int16), cl[keep].view(torch.int16))


def test_obs2_to_nhwc(dev):
    """the two-source stem input bit for bit against torch.cat((obs, inv), 1).to(bfloat16), padding +0.0: every version's oracle
    split and splits whose boundary falls inside a 64-channel chunk, at a chunk edge, or leaves a chunk of padding only"""
    import torch

    from mortal_b200 import nn_ops

    gen = torch.Generator(device="cuda").manual_seed(25)
    splits = ((938, 211, 1152), (942, 217, 1216), (934, 217, 1152), (1012, 217, 1280), (40, 50, 128), (64, 8, 128), (1, 1, 64),
              (70, 3, 192), (5, 100, 128))
    for c1, c2, cpad in splits:
        for l in (1, 34, 128):
            for b in (1, 4099 if c1 + c2 > 200 else 301):
                obs = _special_floats(b * c1 * l, gen).view(b, c1, l)
                inv = _special_floats(b * c2 * l, gen).view(b, c2, l)
                out = nn_ops.obs2_to_nhwc(obs, inv, cpad)
                what = f"obs2_to_nhwc B={b} C1={c1} C2={c2} pad={cpad} L={l}"
                assert out.shape == (b, cpad, 1, l) and out.is_contiguous(memory_format=torch.channels_last), what
                R.check_bits(what, out[:, :c1 + c2, 0, :], torch.cat((obs, inv), 1).to(torch.bfloat16), ("b", "c", "l"))
                assert (out[:, c1 + c2:].contiguous().view(torch.int16) == 0).all(), what
                del obs, inv, out
        torch.cuda.empty_cache()


def test_new_wrappers_refuse_misaligned_tensors(dev, monkeypatch):
    import torch

    from mortal_b200 import _lib, nn_ops

    def no_load():
        raise AssertionError("reached libmjx with a misaligned tensor")

    b, c, l, h = 3, 16, 5, 2
    cl = lambda t: t.contiguous(memory_format=torch.channels_last)
    x = cl(torch.randn(b, c, 1, l, device="cuda").to(torch.bfloat16))
    y = cl(torch.randn(b, c, 1, l, device="cuda").to(torch.bfloat16))
    f32 = lambda *n: torch.rand(*n, device="cuda")
    mis32 = lambda *shape: torch.empty(math.prod(shape) + 1, device="cuda")[1:].view(*shape)
    base = torch.empty(b * l * c + 8, dtype=torch.bfloat16, device="cuda")
    mis_x = base[1:1 + b * l * c].view(b, l, c).permute(0, 2, 1).unsqueeze(2)
    monkeypatch.setattr(_lib, "load", no_load)
    cases = [lambda: nn_ops.affine_relu(mis_x, f32(c), f32(c)), lambda: nn_ops.affine_relu(x, mis32(c), f32(c)),
             lambda: nn_ops.affine_relu(x, f32(c), mis32(c))]
    tail = dict(y=y, x=x, scale=f32(c), bias=f32(c), w1=f32(h, c), b1=f32(h), w2t=f32(h, c), b2=f32(c))
    for k in tail:
        bad = dict(tail)
        bad[k] = mis_x if k in ("y", "x") else mis32(*tail[k].shape)
        cases.append(lambda bad=bad: nn_ops.post_block_tail(**bad))
    for i, case in enumerate(cases):
        with pytest.raises(AssertionError, match="16-byte|channels_last") as e:
            case()
        assert "reached libmjx" not in str(e.value), i


# ---- networks ------------------------------------------------------------------------------------------------------------------

def _random_bn(brain):
    import torch

    for m in brain.modules():
        if isinstance(m, torch.nn.BatchNorm1d):
            m.running_mean.normal_(0, 0.1); m.running_var.uniform_(0.5, 1.5); m.weight.data.uniform_(0.5, 1.5); m.bias.data.normal_(0, 0.1)
    return brain


@pytest.fixture(scope="module")
def arena_rows(dev):
    """real decision rows of 128 tables fast-forwarded 120 steps: (env, rows), the env kept open for other obs versions"""
    import torch

    import mortal_b200

    n = 128
    env = mortal_b200.BatchEnv(np.repeat(np.arange(20000, 20000 + n // 4, dtype=np.uint64), 4), np.full(n, 0x2000, dtype=np.uint64))
    actions = torch.zeros(env.row_cap, dtype=torch.int64, device=env.device)
    env.step(None)
    for _ in range(120):
        env.policy_test(1, actions)
        env.step(actions)
    nr = env.num_rows()
    assert nr >= 64
    rows = {}
    for v in (1, 2, 3, 4):
        env.set_obs_version(v)
        rows[v] = (env.encode_obs()[:nr].clone(), env.encode_invisible(v)[:nr].clone())
    masks = env.masks[:nr].clone().bool()
    env.close()
    return rows, masks


def test_v1_and_v4_oracle_layer_by_layer(dev, arena_rows):
    """Brain(192, 40) of version 1 and the version-4 oracle brain, walked the way forward_fast runs them: every fused kernel and
    every convolution against float64 of that layer's inputs, the walk's output equal to forward_fast bit for bit"""
    import torch

    F = torch.nn.functional
    from mortal_b200 import nn_ops
    from mortal_b200.model import Brain
    from test_gpu_nn_numerics import call_block_tail, check_affine_mish, check_block_tail

    rows, _ = arena_rows
    for version, oracle in ((1, False), (4, True)):
        torch.manual_seed(31 + version)
        brain = _random_bn(Brain(conv_channels=192, num_blocks=40, version=version, is_oracle=oracle)).to(dev).eval()
        with torch.no_grad():
            brain.prepare_fast(torch.bfloat16)
        obs, inv = rows[version]
        inv = inv if oracle else None
        conv = ConvStats()
        what = f"v{version}{' oracle' if oracle else ''}"
        with torch.inference_mode():
            if oracle:
                xin = nn_ops.obs2_to_nhwc(obs, inv, brain._cpad)
                R.check_bits(f"{what} stem input", xin[:, :obs.shape[1] + inv.shape[1], 0], torch.cat((obs, inv), 1).to(torch.bfloat16))
            else:
                xin = nn_ops.obs_to_nhwc(obs, brain._cpad)
            x = F.conv2d(xin, brain._w_stem_pad, padding=(0, 1))
            conv.check(f"{what} stem conv", xin, brain._w_stem_pad, x)
            n = len(brain.blocks)
            if version == 1:
                f, g = brain._aff32_out
                a = call_affine_relu(x, f, g)
                check_affine_relu(x, f, g, a, f"{what} stem bn")
                x = a
                for i in range(n):
                    (w1, w2), ((f1, g1), (f2, g2)) = brain._w[i], brain._aff32[i]
                    y = F.conv2d(x, w1, padding=(0, 1))
                    conv.check(f"{what} block {i} conv1", x, w1, y)
                    a = call_affine_relu(y, f1, g1)
                    check_affine_relu(y, f1, g1, a, f"{what} block {i} bn1")
                    y2 = F.conv2d(a, w2, padding=(0, 1))
                    conv.check(f"{what} block {i} conv2", a, w2, y2)
                    gate, x_new = call_post_tail(y2, x, f2, g2, *brain._gate32[i])
                    check_post_tail(y2, x, f2, g2, brain._gate32[i], gate, x_new, f"{what} block {i} tail")
                    x = x_new
                c = F.conv2d(x, brain._w_neck, brain.neck.bias, padding=(0, 1))
                conv.check(f"{what} neck conv", x, brain._w_neck, c, brain.neck.bias)
                latent = F.relu(brain.latent(brain.fc(F.relu(c).flatten(1))))
                walk = (brain.mu_head(latent), brain.logsig_head(latent))
            else:
                f, g = brain._aff32[0][0]
                a = nn_ops.affine_mish(x, f, g)
                check_affine_mish(x, f, g, a, f"{what} block 0 bn1")
                for i in range(n):
                    (w1, w2), (_, (f2, g2)) = brain._w[i], brain._aff32[i]
                    y = F.conv2d(a, w1, padding=(0, 1))
                    conv.check(f"{what} block {i} conv1", a, w1, y)
                    a2 = nn_ops.affine_mish(y, f2, g2)
                    check_affine_mish(y, f2, g2, a2, f"{what} block {i} bn2")
                    y2 = F.conv2d(a2, w2, padding=(0, 1))
                    conv.check(f"{what} block {i} conv2", a2, w2, y2)
                    nf, ng = brain._aff32[i + 1][0] if i + 1 < n else brain._aff32_out
                    gate, x_new, a = call_block_tail(y2, x, *brain._gate32[i], nf, ng)
                    check_block_tail(y2, x, brain._gate32[i], nf, ng, gate, x_new, a, f"{what} block {i} tail")
                    x = x_new
                c = F.conv2d(a, brain._w_neck, brain.neck.bias, padding=(0, 1))
                conv.check(f"{what} neck conv", a, brain._w_neck, c, brain.neck.bias)
                walk = (F.mish(brain.fc(F.mish(c).flatten(1))),)
            fast = brain.forward_fast(obs, inv)
            fast = fast if isinstance(fast, tuple) else (fast,)
        print(f"{what}: conv max |got - v| / sum|w a| = {conv.rel:.3g}, share of the accumulation term {conv.share:.3g}")
        for w, f in zip(walk, fast):
            assert torch.equal(w.view(torch.int16), f.view(torch.int16)), f"{what}: the walk is not the production composition"
        assert conv.share <= 0.25, (what, conv.share)
        del brain
        torch.cuda.empty_cache()


def _engines(dev, **kw):
    """a DeviceEngine per fixture case, loaded from its checkpoint"""
    import mortal_ckpt as K
    from mortal_b200.engine import DeviceEngine
    from mortal_b200.model import load_mortal

    fx = K.load_fixture()
    out = {}
    for name, (version, oracle, _) in K.CASES.items():
        brain, dqn = load_mortal(K.checkpoint(name, fx[name]))
        out[name] = DeviceEngine(brain, dqn, version=version, is_oracle=oracle, device=dev, name=name, **kw)
    return out


def test_every_version_end_to_end_on_arena_rows(dev, arena_rows):
    """per checkpoint: the fused engine's legal Q-values against the float64 stock forward of the same weights on real arena rows,
    max |dq| relative to the largest |q|. A plain version may show at most twice the error of the version-4 path (the one bench
    runs) on the same rows. An oracle brain reads rows the version-4 path does not take (the invisible observation on top), so its
    yardstick is the same network's stock module under bf16 autocast on the same rows (what DeviceEngine runs for a module without
    the fast path): the fused path may show at most twice that error."""
    import torch

    rows, masks = arena_rows
    errs = {}
    for name, eng in _engines(dev).items():
        obs, inv = rows[eng.version]
        extra = (inv,) if eng.is_oracle else ()
        _, q = eng.react_device(obs, masks, invisible_obs=inv if eng.is_oracle else None)
        with torch.inference_mode():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                q_amp = eng.dqn(eng._latent(eng.brain(obs, *extra)), masks).float()
            qref = eng.dqn.double()(eng._latent(eng.brain.double()(obs.double(), *(t.double() for t in extra))), masks)
        eng.brain.float(), eng.dqn.float()
        top = qref[masks].abs().max().item()
        errs[name] = tuple((d.double() - qref)[masks].abs().max().item() / top for d in (q, q_amp))
    print("max |dq| / max |q| (fused, stock under autocast):", {k: (f"{a:.3g}", f"{b:.3g}") for k, (a, b) in errs.items()})
    for name, (fused, amp) in errs.items():
        bound = 2 * amp if name.endswith("oracle") else 2 * errs["v4"][0]
        assert fused <= bound, (name, errs)


def test_react_static_equals_react_device_every_version(dev):
    """the CUDA-graph replay is bit-identical to the eager forward for each non-oracle version"""
    import torch

    from mortal_b200.model import OBS_ROWS

    for name, eng in _engines(dev).items():
        if eng.is_oracle:
            continue
        gen = torch.Generator(device="cuda").manual_seed(eng.version)
        obs = (torch.rand(600, OBS_ROWS[eng.version], 34, generator=gen, device="cuda") < 0.05).float()
        masks = torch.rand(600, 46, generator=gen, device="cuda") > 0.5
        masks[:, 45] = True
        for nr in (300, 600):
            nb = min(-(-nr // 256) * 256, 600)
            a0, q0 = eng.react_device(obs[:nb], masks[:nb])
            a1, q1 = eng.react_static(obs, masks, nr)
            assert torch.equal(a0[:nr], a1) and torch.equal(q0[:nr].view(torch.int32), q1.view(torch.int32)), (name, nr)
        assert eng._graphs, name


def test_checkpoint_engines_play_the_arena(dev):
    """each checkpoint-loaded engine plays OneVsThree against the version-4 one; the recorded decisions replay in the oracle to
    the same scores and ranks"""
    import mortal_b200.libriichi as lr
    import oracle_lib as O

    lr.install()
    from libriichi.arena import OneVsThree

    engines = _engines(dev)
    seed_count = 3
    for name, eng in engines.items():
        arena = OneVsThree(disable_progress_bar=True, log_dir=None)
        arena.record_decisions = True
        seed_start = (30000 + 10 * eng.version + eng.is_oracle, 0x2000)
        rankings = arena.py_vs_py(challenger=eng, champion=engines["v4"] if name != "v4" else eng, seed_start=seed_start,
                                  seed_count=seed_count)
        assert sum(rankings) == 4 * seed_count, name
        n = 4 * seed_count
        nonces = np.repeat(np.arange(seed_start[0], seed_start[0] + seed_count, dtype=np.uint64), 4)
        ref = O.run_replay(nonces, np.full(n, seed_start[1], dtype=np.uint64), arena.last_decisions, quick_eval=True)
        got = arena.last_results
        assert (got["scores"] == ref["scores"]).all() and (got["ranks"] == ref["ranks"]).all(), name


def test_v1_oracle_engine_gets_its_own_invisible_rows(dev):
    """a version-1 oracle engine facing a version-4 engine receives 211-row invisible observations, each equal to a row of the
    environment's version-1 invisible encoding of the same state"""
    import torch

    import mortal_b200
    import mortal_b200.libriichi as lr

    lr.install()
    from libriichi.arena import OneVsThree

    engines = _engines(dev)
    envs, calls = [], []

    class Env(mortal_b200.BatchEnv):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            envs.append(self)

    class Spy:
        def __init__(self, eng):
            self.eng = eng
            for a in ("name", "version", "is_oracle", "enable_quick_eval", "enable_rule_based_agari_guard"):
                setattr(self, a, getattr(eng, a))

        def react_device(self, obs, masks, invisible_obs=None):
            assert invisible_obs is not None and invisible_obs.shape[1:] == (211, 34) and obs.shape[1:] == (938, 34)
            got = invisible_obs.clone()
            env = envs[-1]
            full = env.encode_invisible(1)[:env.num_rows()].clone()
            calls.append(bool(((got[:, None] == full[None]).flatten(2).all(-1)).any(1).all()))
            return self.eng.react_device(obs, masks, invisible_obs=got)

    arena = OneVsThree(disable_progress_bar=True, log_dir=None)
    arena.env_factory = Env
    arena.max_cycles = 60
    arena.py_vs_py(challenger=Spy(engines["v1_oracle"]), champion=engines["v4"], seed_start=(40000, 0x2000), seed_count=2)
    assert len(calls) > 10 and all(calls), calls


def test_two_vs_two_between_versions(dev):
    """a version-1 and a version-3 engine play TwoVsTwo to the end"""
    import mortal_b200.libriichi as lr

    lr.install()
    from libriichi.arena import TwoVsTwo

    engines = _engines(dev)
    arena = TwoVsTwo(disable_progress_bar=True, log_dir=None)
    arena.py_vs_py(challenger=engines["v1"], champion=engines["v3"], seed_start=(50000, 0x2000), seed_count=2)
    res = arena.last_results
    assert (res["done"] == 1).all() and (res["err"] == 0).all() and (res["steps"] > 0).all()
