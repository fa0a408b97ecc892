"""mortal.py: the mjai bot end users run, for one seat.

    python -m mortal_b200.mortal ID                          live play: every stdin line to libriichi.mjai.Bot, its reactions out
    MORTAL_REVIEW_MODE=1 python -m mortal_b200.mortal ID     review: all of stdin is one log; prints review.review_logs' text

The config comes from MORTAL_CFG (train_grp.load_config): control.state_file is the checkpoint, [grp] network / state_file the GRP
the review's extra_data line needs. The engine is built as mortal.py builds it (fp32 DeviceEngine, TF32 off, no quick eval in
review mode, the rule-based agari guard on), so its Q-values are the reference's fp32 ones up to summation order.
"""
from __future__ import annotations

import os
import sys
from datetime import datetime, timezone

USAGE = """Usage: python -m mortal_b200.mortal <ID>

ARGS:
    <ID>    The player ID, an integer within [0, 3]."""


def model_tag(state: dict) -> str:
    if "tag" in state:
        return state["tag"]
    cfg = state["config"]
    version = cfg["control"].get("version", 1)
    time = datetime.fromtimestamp(state["timestamp"], tz=timezone.utc).strftime("%y%m%d%H")
    return f"mortal{version}-b{cfg['resnet']['num_blocks']}c{cfg['resnet']['conv_channels']}-t{time}"


def load_engine(review_mode: bool, config=None):
    """(DeviceEngine, the checkpoint) as mortal.py builds its engine from config['control']['state_file']"""
    import torch

    from .engine import DeviceEngine
    from .model import load_mortal
    from .train_grp import load_config

    config = config or load_config()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    state = torch.load(config["control"]["state_file"], weights_only=True, map_location="cpu")
    brain, dqn = load_mortal(state)
    engine = DeviceEngine(brain, dqn, version=state["config"]["control"].get("version", 1), is_oracle=False, enable_amp=False,
                          enable_quick_eval=not review_mode, enable_rule_based_agari_guard=True, name="mortal")
    return engine, state


def load_review_engine(config=None):
    """(engine, GRP state dict, model tag) of a review, from the config"""
    import torch

    from .train_grp import load_config

    config = config or load_config()
    engine, state = load_engine(True, config)
    grp_state = torch.load(config["grp"]["state_file"], weights_only=True, map_location="cpu")
    return engine, grp_state["model"], model_tag(state)


def main(argv=None) -> int:
    argv = sys.argv[1:] if argv is None else argv
    try:
        player_id = int(argv[-1])
        assert player_id in range(4)
    except Exception:  # noqa: BLE001 — any bad argument: the usage
        print(USAGE, file=sys.stderr)
        return 1
    if os.environ.get("MORTAL_REVIEW_MODE", "0") == "1":
        from .review import review_logs

        engine, grp, tag = load_review_engine()
        (r,), = review_logs(engine, [sys.stdin.read()], [player_id], grp=grp, model_tag=tag)
        if r.error is not None:
            print(r.error, file=sys.stderr)
            return 1
        sys.stdout.write(r.text)
        sys.stdout.flush()
        return 0
    from .libriichi.mjai import Bot

    engine, _ = load_engine(False)
    bot = Bot(engine, player_id)
    for line in sys.stdin:
        line = line.strip()
        if line and (reaction := bot.react(line)):
            print(reaction, flush=True)
    return 0


if __name__ == "__main__":
    try:
        sys.exit(main())
    except KeyboardInterrupt:
        pass
