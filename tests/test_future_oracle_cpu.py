"""CPU: the future-prediction oracle (oracle/future_oracle.py) reproduces, bit for bit, what the reference's FuturePrediction and
SpatialGRU computed when oracle/gen_golden_future.py recorded tests/golden/future_prediction.npz: outputs, input and state
gradients, every parameter gradient and the running statistics after a train step, in train and eval mode."""
import os

import numpy as np
import pytest
import torch

from oracle import future_oracle as FO
from oracle.gen_golden_future import step
from tests.conftest import GOLDEN_DIR


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN_DIR, "future_prediction.npz"))


def _model(name):
    return FO.FuturePrediction(8, 4) if name == "future" else FO.SpatialGRU(5, 6, gru_bias_init=0.25)


@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("name", ["future", "gru"])
def test_oracle_matches_the_reference(golden, name, train):
    model = _model(name)
    sd = {k[len(f"{name}__sd__"):]: torch.from_numpy(golden[k]) for k in golden.files if k.startswith(f"{name}__sd__")}
    assert list(sd) == list(model.state_dict())
    model.load_state_dict(sd)
    x, h0, gout = (torch.from_numpy(golden[f"{name}__{k}"]) for k in ("x", "h0", "gout"))
    got = step(model, x, h0, gout, train)
    tag = f"{name}__{'train' if train else 'eval'}__"
    want = [k for k in golden.files if k.startswith(tag)]
    assert sorted(k[len(tag):] for k in want) == sorted(got)
    for k in want:
        assert np.array_equal(got[k[len(tag):]].numpy(), golden[k]), k
