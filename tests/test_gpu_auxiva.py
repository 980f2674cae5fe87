"""
GPU tier of AuxIVA (setk_auxiva_stft on the H100): full-size parity with the float64 oracle,
the reference fixtures, run-to-run bit identity and the apply_auxiva.py command line.
"""
import numpy as np
import pytest
import torch

import auxiva_cases as ac

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("N", [4, 8])
def test_fullsize_vs_float64_oracle(cuda, N):
    """B = 16 utterances of 10 s (T = 626, F = 257), 20 epochs; first and last utterance checked."""
    ac.run_parity(cuda, 16, N, 257, 626, 20, np.random.default_rng(40 + N), check=(0, 15))


def test_reference_fixtures(cuda):
    ac.run_fixtures(cuda)


def test_two_calls_bit_identical(cuda):
    from setk_b200 import plan
    X = torch.from_numpy(ac.mixture(np.random.default_rng(9), 8, 4, 257, 300)).to(cuda)
    Y1, s1 = plan.auxiva_from_stft(X, num_epochs=20)
    Y2, s2 = plan.auxiva_from_stft(X, num_epochs=20)
    assert torch.equal(torch.view_as_real(Y1), torch.view_as_real(Y2)) and torch.equal(s1, s2)


def test_apply_auxiva_cli(tmp_path, cuda):
    ac.check_cli(tmp_path)
