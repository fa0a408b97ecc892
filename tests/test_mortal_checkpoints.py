"""Mortal checkpoints of every version load into mortal_b200.model and compute what the reference's networks compute
(tests/golden/mortal_model_outputs.npz, made by tools/extract_model_fixtures.py from the reference's own mortal/model.py); the
fast path in fp32 is the same function; the loader refuses what does not fit; the new libmjx entries check their pointers."""
import copy
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import mortal_ckpt as K
from mortal_b200.model import DQN, Brain, load_mortal


@pytest.fixture(scope="module")
def fx():
    return K.load_fixture()


def _inputs(name, fx, dtype):
    d = fx[name]
    version, is_oracle, seed = K.CASES[name]
    unpack = lambda a: torch.from_numpy(np.unpackbits(a, axis=-1, count=34).astype(np.float32)).to(dtype)
    obs = unpack(d["obs"])
    inv = unpack(d["inv"]) if is_oracle else None
    o2, i2, m2 = K.observations(version, is_oracle, seed)  # the stored batch is the seeded one
    assert np.array_equal(obs.float().numpy(), o2) and np.array_equal(d["masks"], m2)
    return obs, inv, torch.from_numpy(d["masks"])


def _rel(got, ref):
    ref = torch.as_tensor(ref, dtype=torch.float64)
    return ((got.double() - ref).abs().max() / ref.abs().max()).item()


@pytest.mark.parametrize("name", list(K.CASES))
def test_load_mortal_equals_reference_in_float64(name, fx):
    version, is_oracle, _ = K.CASES[name]
    brain, dqn = load_mortal(K.checkpoint(name, fx[name]))
    assert (brain.version, brain.is_oracle, dqn.version) == (version, is_oracle, version) and not brain.training
    brain, dqn = brain.double(), dqn.double()
    obs, inv, masks = _inputs(name, fx, torch.float64)
    with torch.no_grad():
        out = brain(obs, inv)
        if version == 1:
            assert _rel(out[0], fx[name]["mu"]) < 1e-12 and _rel(out[1], fx[name]["logsig"]) < 1e-12
            phi = out[0]
        else:
            phi = out
            assert _rel(phi, fx[name]["phi"]) < 1e-12
        q = dqn(phi, masks)
    ref_q = torch.from_numpy(fx[name]["q"])
    assert torch.equal(torch.isinf(q), torch.isinf(ref_q)) and torch.isinf(q[~masks]).all()
    assert _rel(q[masks], ref_q[masks]) < 1e-12


@pytest.mark.parametrize("name", list(K.CASES))
def test_prepare_fast_fp32_equals_stock_forward(name, fx):
    brain, _ = load_mortal(K.checkpoint(name, fx[name]))
    obs, inv, _ = _inputs(name, fx, torch.float32)
    fast = copy.deepcopy(brain)
    with torch.no_grad():
        ref = brain(obs, inv)
        fast.prepare_fast(None)
        got = fast.forward_fast(obs, inv)
    ref, got = (ref, got) if isinstance(ref, tuple) else ((ref,), (got,))
    for r, g in zip(ref, got):
        assert r.shape == g.shape and (r - g).abs().max() <= 1e-5 * max(1.0, r.abs().max().item())


def test_reference_key_layout_is_the_fixture_layout(fx):
    """the keys load_mortal expects are exactly the reference's state-dict keys, in the reference's order"""
    from mortal_b200.model import _reference_prefixes

    for name, (version, is_oracle, _) in K.CASES.items():
        b = Brain(conv_channels=K.CONV_CHANNELS, num_blocks=K.NUM_BLOCKS, version=version, is_oracle=is_oracle)
        names = _reference_prefixes(b)
        mine = [(names[k.rsplit(".", 1)[0]] + "." + k.rsplit(".", 1)[1], list(t.shape)) for k, t in b.state_dict().items()]
        assert sorted(map(list, mine)) == sorted(map(list, fx[name]["brain_keys"])), name
        assert [[k, list(t.shape)] for k, t in DQN(version=version).state_dict().items()] == [list(x) for x in fx[name]["dqn_keys"]]


def test_load_mortal_refuses_what_does_not_fit(fx):
    good = K.checkpoint("v4", fx["v4"])
    load_mortal(good)
    some = "encoder.net.2.ca.shared_mlp.0.weight"
    bad = copy.deepcopy(good)
    del bad["mortal"][some]
    with pytest.raises(KeyError, match="missing key 'encoder.net.2.ca.shared_mlp.0.weight'"):
        load_mortal(bad)
    bad = copy.deepcopy(good)
    bad["mortal"]["encoder.net.1.res_unit.9.weight"] = torch.zeros(3)
    with pytest.raises(KeyError, match="unexpected key 'encoder.net.1.res_unit.9.weight'"):
        load_mortal(bad)
    bad = copy.deepcopy(good)
    bad["current_dqn"]["v_head.weight"] = torch.zeros(1, 1024)
    with pytest.raises(KeyError, match="current_dqn: unexpected key 'v_head.weight'"):
        load_mortal(bad)
    bad = copy.deepcopy(good)
    bad["mortal"][some] = torch.zeros(3, 32)
    with pytest.raises(ValueError, match="'encoder.net.2.ca.shared_mlp.0.weight' has shape \\(3, 32\\), expected \\(2, 32\\)"):
        load_mortal(bad)
    for v in (0, 5):
        bad = copy.deepcopy(good)
        bad["config"]["control"]["version"] = v
        with pytest.raises(ValueError, match=f"unsupported Mortal version {v}"):
            load_mortal(bad)
    bad = copy.deepcopy(good)
    bad["mortal"]["encoder.net.0.weight"] = torch.zeros(32, 1013, 3)
    with pytest.raises(ValueError, match="reads 1013 channels, which is neither"):
        load_mortal(bad)
    bad = copy.deepcopy(good)
    bad["config"]["control"]["version"] = 3  # a v4 state dict under a v3 config: 1012 rows fit neither v3 width
    with pytest.raises(ValueError, match="reads 1012 channels"):
        load_mortal(bad)
    bad = copy.deepcopy(good)
    bad["config"]["resnet"]["conv_channels"] = 64
    with pytest.raises(ValueError, match="config resnet.conv_channels is 64"):
        load_mortal(bad)
    bad = copy.deepcopy(good)
    bad["config"]["resnet"]["num_blocks"] = 3
    with pytest.raises(ValueError, match="config resnet.num_blocks is 3"):
        load_mortal(bad)
    # num_batches_tracked is accepted when present and not required
    ok = copy.deepcopy(good)
    for k in [k for k in ok["mortal"] if k.endswith("num_batches_tracked")]:
        del ok["mortal"][k]
    load_mortal(ok)


def _digest(m):
    h = hashlib.sha256()
    for k, t in m.state_dict().items():
        h.update(k.encode()); h.update(str(tuple(t.shape)).encode()); h.update(t.detach().cpu().contiguous().numpy().tobytes())
    return h.hexdigest()


def test_version4_construction_is_unchanged():
    """Brain(version=4) and DQN(version=4) under torch.manual_seed(0): the same modules, creation order and initial values as
    before the other versions were added (digests of the state dicts of that construction), so bench's network is unchanged"""
    want = {(32, 2): ("c27b804be3dfa43abc14695f8f1dc9b12376eeb8f1c068886d73b7c8b384ccb8",
                      "1194fc67b7f905b778e6fe2b3eab97e2fde9e238c423be81f4409decb39c5207"),
            (192, 40): ("ac9b021236320e71e5ca36fe3a620eb6d1c16bcd38413fc94ac672d50e259c44",
                        "9b16d8b35fca1c67e3b21967021ffd28599215a9ecd06a60ea9a999c180e324d")}
    for (c, n), (db, dd) in want.items():
        torch.manual_seed(0)
        b = Brain(conv_channels=c, num_blocks=n, version=4)
        d = DQN(version=4)
        assert (_digest(b), _digest(d)) == (db, dd), (c, n)


C_ENTRY_CHECK = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from mortal_b200 import _lib
L = _lib.load()  # never mjx_init: no entry can launch a kernel, whatever it is handed
A = 1 << 24      # an aligned address; nothing is dereferenced before the argument checks
entries = {
    "affine_relu": (L.mjx_nn_affine_relu_bf16, 4, lambda p: (*p, 8 * 34 * 64, 64, None)),
    "post_block_tail": (L.mjx_nn_post_block_tail_bf16, 10, lambda p: (*p, 8, 34, 64, 4, None)),
    "obs2_to_nhwc": (L.mjx_nn_obs2_to_nhwc_bf16, 3, lambda p: (*p, 8, 1012, 217, 34, 1280, None)),
}
res = {}
for name, (fn, n, args) in entries.items():
    ptrs = [A + 4096 * i for i in range(n)]
    res[name] = {"aligned": fn(*args(ptrs)),
                 "misaligned": [fn(*args([q + (4 if j == i else 0) for j, q in enumerate(ptrs)])) for i in range(n)]}
    if name == "obs2_to_nhwc":  # the observations need float alignment only
        res[name]["float_aligned"] = [fn(*args([ptrs[0] + 4, ptrs[1], ptrs[2]])), fn(*args([ptrs[0], ptrs[1] + 4, ptrs[2]]))]
        res[name]["misaligned"][:2] = [fn(*args([ptrs[0] + 2, ptrs[1], ptrs[2]])), fn(*args([ptrs[0], ptrs[1] + 2, ptrs[2]]))]
        res[name]["too_narrow"] = fn(*(ptrs + [8, 1012, 217, 34, 1216, None]))
print(json.dumps(res))
"""


def test_new_c_entries_refuse_misaligned_pointers_before_state():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", C_ENTRY_CHECK, root], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-3000:]
    res = json.loads(out.stdout.strip().splitlines()[-1])
    ERR_ARG, ERR_STATE = -2, -4
    for name, r in res.items():
        assert r["aligned"] == ERR_STATE, (name, r)
        assert r["misaligned"] == [ERR_ARG] * len(r["misaligned"]), (name, r)
    assert res["obs2_to_nhwc"]["float_aligned"] == [ERR_STATE, ERR_STATE]
    assert res["obs2_to_nhwc"]["too_narrow"] == ERR_ARG  # 1012 + 217 channels do not fit 1216
