"""CPU: the decoder oracle's ``output_head`` (oracle/decoder_oracle.py) reproduces, bit for bit, what the reference's four output heads of
a ``Decoder(16, 3, True)`` computed when oracle/gen_golden_decoder.py recorded tests/golden/decoder_heads.npz: the output, the input
gradient, every parameter gradient and the buffers after a step, in train and eval mode.  The restatement of
tests/_output_head_cases.py and the module tests of the kernels trust this head."""
import os

import numpy as np
import pytest
import torch

from oracle import decoder_oracle as DO
from oracle.gen_golden_decoder import HEADS, HEAD_CHANNELS, head_step
from tests.conftest import GOLDEN_DIR


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN_DIR, "decoder_heads.npz"))


@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("name,n_out,sigmoid", HEADS, ids=[h[0] for h in HEADS])
def test_output_head_matches_the_reference(golden, name, n_out, sigmoid, train):
    head = DO.output_head(HEAD_CHANNELS, n_out, sigmoid)
    sd = {k[len(f"{name}__sd__"):]: torch.from_numpy(golden[k]) for k in golden.files if k.startswith(f"{name}__sd__")}
    assert list(sd) == list(head.state_dict())
    head.load_state_dict(sd)
    x, gout = (torch.from_numpy(golden[f"{name}__{k}"]) for k in ("x", "gout"))
    got = head_step(head, x, gout, train)
    tag = f"{name}__{'train' if train else 'eval'}__"
    want = [k for k in golden.files if k.startswith(tag)]
    assert sorted(k[len(tag):] for k in want) == sorted(got)
    for k in want:
        assert np.array_equal(got[k[len(tag):]].numpy(), golden[k]), k
