"""
GPU tier of noise suppression (setk_ns_imcra on the H100): full-size parity with the float64
oracle, the reference's gains on the doc clip and the stored cases, run-to-run bit identity and
the apply_ns.py command line.
"""
import numpy as np
import pytest
import torch

import ns_cases as nc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("F", [257, 513])
def test_fullsize_vs_float64_oracle(cuda, F):
    """B = 16 utterances of 10 s at hop 256 (T = 626), n_fft 512 and 1024; first and last checked."""
    nc.run_parity(cuda, 16, F, 626, {}, np.random.default_rng(50 + F), check=(0, 15))


def test_fullsize_ragged_case_b(cuda):
    n_frames = [626, 313, 1, 600]
    nc.run_parity(cuda, 4, 257, 626, nc.CASE_B_CONF, np.random.default_rng(8), n_frames=n_frames)


def test_reference_clip(cuda):
    nc.run_clip(cuda)


def test_reference_cases(cuda):
    nc.run_cases(cuda)


def test_two_calls_bit_identical(cuda):
    from setk_b200 import plan
    X = torch.from_numpy(nc.noisy_stft(np.random.default_rng(9), 8, 513, 300)).to(cuda)
    g1, e1 = plan.ns_from_stft(X)
    g2, e2 = plan.ns_from_stft(X)
    assert torch.equal(g1, g2) and torch.equal(torch.view_as_real(e1), torch.view_as_real(e2))


def test_largest_fft_runs(cuda):
    """n_fft 4096 (F = 2049): five bins per thread."""
    nc.run_parity(cuda, 2, 2049, 40, {}, np.random.default_rng(10), check=(1,))


def test_apply_ns_cli(tmp_path, cuda):
    exact = nc.check_cli(tmp_path)
    print(f"apply_ns.py on the H100: {exact:.6f} of the samples equal egs_ns.wav")
