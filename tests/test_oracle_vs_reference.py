"""CPU: the oracle restatement reproduces the REAL reference forward, as stored in tests/golden/reference_cases.npz by
oracle/make_golden_reference_cases.py: state-dict keys and shapes exactly; 1024 strided logits within fp32 reduction-order
noise; the argmax map on every pixel whose class margin exceeds 1e-4."""
import os

import numpy as np
import pytest

from oracle import dinounet_oracle as O
from oracle.make_golden_reference_cases import sha

REF = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_cases.npz"))


def _check(y, key):
    f = y.reshape(-1)
    samp = f[:: max(1, f.size // 1024)][:1024]
    assert np.abs(samp - REF[key]).max() <= 2e-5
    am = np.unpackbits(REF[key + "_argmax"])[: y.shape[0] * y.shape[2] * y.shape[3]].reshape(y.shape[0], *y.shape[2:])
    margin = np.abs(y[:, 0] - y[:, 1])
    assert ((y.argmax(1) != am) & (margin > 1e-4)).sum() == 0


@pytest.mark.parametrize("model,size", [("dinounet_s", 128), ("dinounet_b", 64), ("dinounet_7b_tiny", 64)])
def test_matches_reference_forward(model, size):
    sd = O.make_state_dict(model, 2, seed=3)
    assert np.array_equal(sha(sorted([k, list(t.shape)] for k, t in sd.items())), REF[f"spec_{model}"])
    yo = O.forward(sd, model, O.make_input(2, size, 5)).numpy()
    assert yo.shape == (2, 2, size, size)
    _check(yo, f"fwd_{model}")


def test_single_channel_input_path():
    """dinounet_training.py:491-497 channel fix-up."""
    sd = O.make_state_dict("dinounet_s", 2, seed=3)
    yo = O.forward(sd, "dinounet_s", O.make_input(1, 64, 7, channels=1)).numpy()
    assert yo.shape == (1, 2, 64, 64)
    _check(yo, "fwd_single_channel")
