"""
CACGMM mask estimation and permutation alignment on the H100: the kernels against the oracle at 1-2 s
utterances, the aligner against the host permu_aligner, every run of the reference's fixture, bit
identity from run to run, and the command line.
"""
import numpy as np
import pytest
import torch

import cacgmm_cases as cc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("C,K,start,fl", [
    (2, 2, "cgmm", 512),
    (2, 4, "random", 512),
    (4, 3, "random", 512),
    (4, 2, "cgmm", 1024),
    (7, 2, "random", 512),
    (7, 4, "random", 1024),
    (9, 3, "random", 512),
    (16, 2, "cgmm", 512),
    (16, 4, "random", 512),
])
def test_kernels_vs_oracle(cuda, C, K, start, fl):
    rng = np.random.default_rng(300 + 10 * C + K)
    cc.check_cacgmm(cuda, rng, 2, C, 32000, fl, K, 8, start, update_alpha=(K != 3),
                    n_samples=[32000, 17000], permu=True)


@pytest.mark.parametrize("F,K", [(257, 2), (257, 3), (257, 4), (513, 2), (513, 3), (513, 4)])
def test_aligner_restores_scrambled_masks(cuda, F, K):
    rng = np.random.default_rng(7 * F + K)
    cc.check_aligner(cuda, cc.scrambled_masks(rng, 3, K, 180, F), n_frames=[180, 121, 64])


def test_aligner_long_utterance_centroids_in_global_memory(cuda):
    """K x T centroids past the shared-memory budget go to global scratch."""
    rng = np.random.default_rng(99)
    cc.check_aligner(cuda, cc.scrambled_masks(rng, 1, 4, 5200, 513))


def test_aligner_on_em_outputs(cuda):
    from setk_b200 import plan as P
    rng = np.random.default_rng(41)
    import parity_cases as pc
    x = torch.from_numpy(pc.structured_audio(rng, 2, 6, 32000)).to(cuda)
    pl = P.StftPlan(6, 512, 256, True, True, "hann", 2, 32000, cuda)
    T, F = pl.num_frames(32000), pl.num_bins
    g = rng.uniform(size=(2, 3, T, F))
    g /= g.sum(1, keepdims=True)
    m, _ = pl.cacgmm_masks(x, 3, 10, init_gamma=torch.from_numpy(g).to(cuda))
    pl.close()
    cc.check_aligner(cuda, m.cpu().numpy().astype(np.float64))


@pytest.mark.parametrize("name", sorted(["2spk", "noisy", "nopermu", "fixed_alpha", "init_mask", "two_utts", "skip"]))
def test_reference_fixture(cuda, name):
    """Every fixture run: the kernels on the reference's STFT within mean 1e-5 / max 5e-3 of its masks, and
    from audio equal to the oracle on the tile STFT; the from-audio distance to the reference is printed."""
    g = cc.fixture()
    assert name in cc.fixture_runs(g)
    cc.check_fixture_reference_stft(cuda, g, name)
    print(name, "from audio vs reference (mean, max):", cc.check_from_audio(cuda, g, name))


def test_run_to_run_bit_identity(cuda):
    from setk_b200 import plan as P
    import parity_cases as pc
    rng = np.random.default_rng(8)
    x = torch.from_numpy(pc.structured_audio(rng, 3, 7, 24000)).to(cuda)
    ns = torch.tensor([24000, 20000, 9000], dtype=torch.int32, device=cuda)
    pl = P.StftPlan(7, 512, 256, True, True, "hann", 3, 24000, cuda)
    T, F = pl.num_frames(24000), pl.num_bins
    g = torch.from_numpy(rng.uniform(size=(3, 3, T, F))).to(cuda)
    g /= g.sum(1, keepdim=True)
    runs = [pl.cacgmm_masks(x, 3, 12, init_gamma=g, permu_plan=P.PERMU_PLANS[F], n_samples=ns)[0].cpu().numpy()
            for _ in range(2)]
    pl.close()
    assert np.array_equal(runs[0], runs[1])


@pytest.mark.parametrize("name", ["2spk", "noisy", "two_utts", "init_mask", "skip"])
def test_cli(cuda, tmp_path, name):
    from setk_b200 import _lib
    cc.run_cli_case(cc.fixture(), name, str(tmp_path), _lib.DEFAULT_LIBRARY, cuda)
