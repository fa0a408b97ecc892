"""mortal_b200.review / mortal_b200.mortal host-side rules (CPU only): which engines a review takes, and the model tag."""
import pytest

import review_lib
from mortal_b200 import mortal, review


def test_review_rejects_oracle_and_quick_eval_engines():
    review.check_engine(review_lib.StubEngine(True))
    quick = review_lib.StubEngine(True)
    quick.enable_quick_eval = True
    oracle = review_lib.StubEngine(False)
    oracle.is_oracle = True
    other = review_lib.StubEngine(False)
    other.engine_type = "other"
    for e in (quick, oracle, other):
        with pytest.raises(ValueError):
            review.review_logs(e, ["{}"], [0])


def test_model_tag():
    cfg = {"control": {"version": 4}, "resnet": {"num_blocks": 40, "conv_channels": 192}}
    assert mortal.model_tag({"tag": "x", "config": cfg}) == "x"
    assert mortal.model_tag({"timestamp": 1700000000, "config": cfg}) == "mortal4-b40c192-t23111422"
    assert mortal.model_tag({"timestamp": 0, "config": {"control": {}, "resnet": cfg["resnet"]}}) == "mortal1-b40c192-t70010100"


def test_mask_eval():
    assert review_lib.mask_eval('{"eval_time_ns":123,"x":{"eval_time_ns":9}}') == '{"eval_time_ns":0,"x":{"eval_time_ns":0}}'
