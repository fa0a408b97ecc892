#!/usr/bin/env python
"""Extract the reference's own test fixtures (data only) into tests/golden/.

usage: python tools/extract_ref_fixtures.py <Mortal checkout>. Outputs are committed:
  tests/golden/state_test_logs.json — the inline mjai JSON logs of libriichi/src/state/test.rs,
      keyed by test fn name, in source order (assert logic is re-stated in tests/test_oracle_state.py)
  tests/golden/golden_game.jsonl — the seeded full-game log embedded in log-viewer/index.example.html:10-264
  tests/golden/tables/*.bin.gz — libriichi/src/algo/data's lookup tables as shipped (tests/test_tables.py)
  tests/golden/reference_engine_game.json.gz — the reference's own, unmodified mortal/engine.py (MortalEngine) and mortal/model.py
      (Brain 16 ch x 1 block, DQN; torch.manual_seed(0), CPU, fp32) playing one seed of OneVsThree.py_vs_py in this repository's
      arena over the host-emulated environment: per engine call a digest of the observations and masks it was handed and the
      actions it chose, then the recorded decisions and the results (tests/test_host_layer.py). Needs `python
      -c "import __graft_entry__ as g; g.build()"` first.
"""
import gzip
import hashlib
import json
import os
import re
import shutil
import sys

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def main(REF):
    os.makedirs(OUT, exist_ok=True)
    src = open(os.path.join(REF, "libriichi/src/state/test.rs")).read()
    logs = {}
    cur = None
    for m in re.finditer(r'fn (\w+)\(\)|r#"(.*?)"#', src, re.S):
        if m.group(1):
            cur = m.group(1)
            continue
        body = m.group(2)
        lines = [ln.strip() for ln in body.strip().split("\n") if ln.strip()]
        for ln in lines:
            json.loads(ln)
        logs.setdefault(cur, []).append(lines)
    with open(os.path.join(OUT, "state_test_logs.json"), "w") as f:
        json.dump(logs, f, indent=0)
    print({k: [len(x) for x in v] for k, v in logs.items()})

    html = open(os.path.join(REF, "log-viewer/index.example.html")).read()
    m = re.search(r"allActions = `\n(.*?)\n\s*`", html, re.S)
    lines = [ln for ln in m.group(1).split("\n") if ln.strip()]
    for ln in lines:
        json.loads(ln)
    with open(os.path.join(OUT, "golden_game.jsonl"), "w") as f:
        f.write("\n".join(lines) + "\n")
    print("golden game lines:", len(lines))

    os.makedirs(os.path.join(OUT, "tables"), exist_ok=True)
    for name in ("shanten_suhai.bin.gz", "shanten_jihai.bin.gz", "agari.bin.gz"):
        shutil.copyfile(os.path.join(REF, "libriichi/src/algo/data", name), os.path.join(OUT, "tables", name))

    game = json.dumps(reference_engine_game(REF), separators=(",", ":")).encode()
    with open(os.path.join(OUT, "reference_engine_game.json.gz"), "wb") as f:
        f.write(gzip.compress(game, mtime=0))


def rows_digest(obs, masks) -> str:
    """sha256 over the float32 observation rows and bool mask rows one engine call was handed (shared with the test)"""
    h = hashlib.sha256()
    h.update(np.ascontiguousarray(np.stack(obs), dtype=np.float32).tobytes())
    h.update(np.ascontiguousarray(np.stack(masks), dtype=bool).tobytes())
    return h.hexdigest()


def reference_engine_game(REF):
    import importlib

    import torch

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [root, os.path.join(root, "tests")]
    import mortal_b200.libriichi as lr
    from emul_batch_env import EmulBatchEnv

    lr.install()
    sys.path.insert(0, os.path.join(REF, "mortal"))
    ref_model, ref_engine = importlib.import_module("model"), importlib.import_module("engine")
    from libriichi.arena import OneVsThree

    class Recording:
        def __init__(self, engine):
            self.engine, self.calls = engine, []

        def __getattr__(self, name):
            return getattr(self.engine, name)

        def react_batch(self, obs, masks, invisible_obs):
            out = self.engine.react_batch(obs, masks, invisible_obs)
            self.calls.append({"rows_sha256": rows_digest(obs, masks), "actions": [int(a) for a in out[0]]})
            return out

    torch.manual_seed(0)
    mk = lambda name: Recording(ref_engine.MortalEngine(ref_model.Brain(version=4, conv_channels=16, num_blocks=1).eval(),
                                                        ref_model.DQN(version=4).eval(), is_oracle=False, version=4,
                                                        device=torch.device("cpu"), enable_amp=False, enable_quick_eval=True,
                                                        enable_rule_based_agari_guard=False, name=name))
    challenger, champion = mk("challenger"), mk("champion")
    arena = OneVsThree(disable_progress_bar=True)
    arena.env_factory = EmulBatchEnv
    arena.record_decisions = True
    rankings = arena.py_vs_py(challenger=challenger, champion=champion, seed_start=(10000, 0x2000), seed_count=1)
    res = arena.last_results
    return {"seed_start": [10000, 0x2000], "seed_count": 1, "rankings": rankings,
            "calls": {"challenger": challenger.calls, "champion": champion.calls},
            "decisions": arena.last_decisions.tolist(), "decision_masks": arena.last_decision_masks.tolist(),
            "scores": res["scores"].tolist(), "ranks": res["ranks"].tolist(), "steps": res["steps"].tolist()}


if __name__ == "__main__":
    main(sys.argv[1])
