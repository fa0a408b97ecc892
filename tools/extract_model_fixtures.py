#!/usr/bin/env python
"""Pin mortal_b200.model to the reference's networks, as data: tests/golden/mortal_model_outputs.npz.

usage: python tools/extract_model_fixtures.py <Mortal checkout>. For every case of tests/mortal_ckpt.py (versions 1-4, oracle
brains of versions 1 and 4; 32 channels, 2 blocks) the reference's own mortal/model.py Brain and DQN are built, filled with the
deterministic weights of tests/mortal_ckpt.py and run in float64 on the case's seeded observations. The file holds per case the
ordered (key, shape) lists of both state dicts, the observations (bit-packed), invisible observations and masks, and the
outputs: phi, or mu and logsig for version 1, and q. The weights themselves are regenerated from the key lists, not stored.
"""
import importlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main(REF):
    import torch

    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    import mortal_b200.libriichi as lr
    import mortal_ckpt as K

    lr.install()  # the reference's model.py imports libriichi.consts
    sys.path.insert(0, os.path.join(REF, "mortal"))
    ref = importlib.import_module("model")
    out = {}
    for name, (version, is_oracle, seed) in K.CASES.items():
        brain = ref.Brain(conv_channels=K.CONV_CHANNELS, num_blocks=K.NUM_BLOCKS, version=version, is_oracle=is_oracle)
        dqn = ref.DQN(version=version)
        bkeys = [(k, list(t.shape)) for k, t in brain.state_dict().items()]
        dkeys = [(k, list(t.shape)) for k, t in dqn.state_dict().items()]
        brain.load_state_dict(K.state_dict(seed, bkeys))
        dqn.load_state_dict(K.state_dict(seed + 1000, dkeys))
        brain, dqn = brain.double().eval(), dqn.double().eval()
        obs, inv, masks = K.observations(version, is_oracle, seed)
        with torch.no_grad():
            o = torch.from_numpy(obs).double()
            i = None if inv is None else torch.from_numpy(inv).double()
            res = brain(o, i)
            if version == 1:
                mu, logsig = res
                out[f"{name}/mu"], out[f"{name}/logsig"] = mu.numpy(), logsig.numpy()
                phi = mu
            else:
                phi = res
                out[f"{name}/phi"] = phi.numpy()
            out[f"{name}/q"] = dqn(phi, torch.from_numpy(masks)).numpy()
        out[f"{name}/brain_keys"] = np.array(json.dumps(bkeys))
        out[f"{name}/dqn_keys"] = np.array(json.dumps(dkeys))
        out[f"{name}/obs"] = np.packbits(obs.astype(bool), axis=-1)
        if inv is not None:
            out[f"{name}/inv"] = np.packbits(inv.astype(bool), axis=-1)
        out[f"{name}/masks"] = masks
        print(name, "brain keys", len(bkeys), "dqn keys", len(dkeys))
    np.savez_compressed(K.FIXTURE, **out)
    print(K.FIXTURE, os.path.getsize(K.FIXTURE), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
