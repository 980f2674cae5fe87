"""
CACGMM mask estimation and permutation alignment, CPU tier: the oracle against the reference's own
runs (tests/golden/ref_cacgmm.npz), and the kernels through the CPU execution model against the
oracle and the host aligner at small sizes.
"""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import cacgmm_cases as cc
from oracle import cacgmm_oracle as ao
from oracle import stft_oracle as so
from oracle.make_golden_cacgmm import oracle_runs


def test_oracle_pinned_to_reference_masks():
    """With the reference's complex64 observations and start, the oracle reproduces every fixture run
    to float32 storage rounding, alignment decisions included."""
    g = cc.fixture()
    pin = json.load(open(os.path.join(cc.GOLD, "PINNING_cacgmm.json")))["oracle_vs_reference"]
    for name in cc.fixture_runs(g):
        for m, ref in oracle_runs(g, name, ao, so, obs_dtype=np.complex64, start_dtype=np.complex64):
            assert np.max(np.abs(m - ref)) <= 1e-7, name
        assert pin[name]["complex64"]["max"] <= 1e-7


@pytest.mark.parametrize("C,fl,K,start,alpha,ragged", [
    (2, 512, 2, "random", True, False),
    (4, 512, 2, "cgmm", False, True),
    (4, 1024, 3, "random", True, True),
    (9, 512, 2, "cgmm", True, False),
    (9, 512, 3, "random", False, False),
    (2, 1024, 2, "cgmm", True, False),
])
def test_kernels_vs_oracle(emu, C, fl, K, start, alpha, ragged):
    rng = np.random.default_rng(160 + C + K)
    B, N, iters = (1, 2600, 2) if C == 9 else (2, 4600, 3)
    ns = [4600, 3300] if ragged else None
    cc.check_cacgmm(emu, rng, B, C, N, fl, K, iters, start, alpha, n_samples=ns, permu=(C != 9))


def test_num_iters_zero_returns_the_start(emu):
    from setk_b200 import plan as P
    rng = np.random.default_rng(5)
    pl = P.StftPlan(3, 512, 256, True, True, "hann", 1, 3000, emu)
    T, F = pl.num_frames(3000), pl.num_bins
    g = rng.uniform(size=(1, 3, T, F))
    g /= g.sum(1, keepdims=True)
    m, _ = pl.cacgmm_masks(torch.from_numpy(pc_audio(rng, 3, 3000)), 3, 0, init_gamma=torch.from_numpy(g))
    assert np.array_equal(m.numpy(), g.astype(np.float32))
    pl.close()


def pc_audio(rng, C, N):
    import parity_cases as pc
    return pc.structured_audio(rng, 1, C, N)


@pytest.mark.parametrize("F,K", [(257, 2), (257, 3), (513, 4), (513, 2)])
def test_aligner_restores_scrambled_masks(emu, F, K):
    rng = np.random.default_rng(F + K)
    T = 24
    masks = cc.scrambled_masks(rng, 2, K, T, F)
    cc.check_aligner(emu, masks, n_frames=[T, 17])


def test_aligner_on_em_outputs(emu):
    from setk_b200 import plan as P
    rng = np.random.default_rng(21)
    x = pc_audio(rng, 4, 5000)
    pl = P.StftPlan(4, 512, 256, True, True, "hann", 1, 5000, emu)
    T, F = pl.num_frames(5000), pl.num_bins
    g = rng.uniform(size=(1, 3, T, F))
    g /= g.sum(1, keepdims=True)
    m, _ = pl.cacgmm_masks(torch.from_numpy(x), 3, 3, init_gamma=torch.from_numpy(g))
    pl.close()
    cc.check_aligner(emu, m.numpy().astype(np.float64))


def test_cgmm_outputs_unchanged(emu):
    """The CGMM shares the E-step, covariance and factor passes: its outputs keep the parent's bits."""
    want = json.load(open(os.path.join(cc.GOLD, "cgmm_emu_sha256.json")))
    assert cc.cgmm_digests(emu) == want


def test_trainer_follows_the_seed(emu):
    """CacgmmTrainer draws its start in the constructor, as the reference does."""
    from setk_b200.libs import utils
    from setk_b200.libs.cluster import CacgmmTrainer
    utils.set_default_device("cpu")
    rng = np.random.default_rng(3)
    obs = (rng.standard_normal((3, 257, 12)) + 1j * rng.standard_normal((3, 257, 12))).astype(np.complex64)
    np.random.seed(7)
    a = CacgmmTrainer(obs, 3).train(2)
    np.random.seed(7)
    g = np.random.uniform(size=[3, 257, 12])
    ref = ao.cacgmm_posteriors(obs, 3, 2, gamma=g / g.sum(0, keepdims=True))
    assert a.shape == (3, 257, 12) and np.max(np.abs(a - ref)) <= cc.TOL_CACGMM
    b = CacgmmTrainer(obs, 2, cgmm_init=True, update_alpha=False).train(2)
    assert np.max(np.abs(b - ao.cacgmm_posteriors(obs, 2, 2, cgmm_init=True, update_alpha=False))) <= cc.TOL_CACGMM
    with pytest.raises(NotImplementedError):
        CacgmmTrainer(obs, 2, cacgmm="model.pkl")


def test_argument_errors(emu):
    from setk_b200 import _lib
    from setk_b200 import plan as P
    pl = P.StftPlan(2, 512, 256, True, True, "hann", 1, 3000, emu)
    x = torch.zeros((1, 2, 3000))
    T, F = pl.num_frames(3000), 257
    before = _lib.launch_count()
    with pytest.raises(ValueError):
        pl.cacgmm_masks(x, 3, 2)                                       # 3 classes need a start
    with pytest.raises(ValueError):
        pl.cacgmm_masks(x, 2, 2)                                       # no start, no cgmm_init
    with pytest.raises(ValueError):
        pl.cacgmm_masks(x, 5, 2, init_gamma=torch.zeros((1, 5, T, F), dtype=torch.float64))
    with pytest.raises(ValueError):
        pl.cacgmm_masks(x, 2, -1, cgmm_init=True)
    with pytest.raises(ValueError):
        pl.cacgmm_masks(x, 2, 2, init_gamma=torch.zeros((1, 2, T + 1, F), dtype=torch.float64))
    with pytest.raises(ValueError):
        pl.cacgmm_masks(x, 2, 2, cgmm_init=True, permu_plan=[(2, 10, 300)])   # hi > F
    with pytest.raises(ValueError):
        pl.cacgmm_masks(x, 2, 2, cgmm_init=True, permu_plan=[(2, 50, 50)])    # empty band
    with pytest.raises(ValueError):
        P.cacgmm_from_stft(torch.zeros((1, 1, 257, 4), dtype=torch.complex64), 2, 2, cgmm_init=True)   # C = 1
    with pytest.raises(ValueError):
        P.permu_align(np.zeros((2, 5, 100)))                           # the reference's Unsupported num_bins
    with pytest.raises(RuntimeError):
        P.permu_align(np.zeros((5, 257)))                              # not K x T x F
    with pytest.raises(ValueError):
        P.permu_align(np.zeros((5, 4, 257)))                           # 5 classes
    assert _lib.launch_count() == before
    pl.close()
    pl = P.StftPlan(2, 256, 64, True, True, "hann", 1, 3000, emu)
    with pytest.raises(Exception):
        pl.cacgmm_masks(x, 2, 2, cgmm_init=True)                      # n_fft 256: no tile STFT
    pl.close()


def test_cabi_checks(emu):
    """The C-ABI refuses what the Python layer refuses, with the documented codes."""
    from setk_b200 import _lib
    lib = _lib.library()
    buf = torch.zeros(4096, dtype=torch.float64)
    p = ctypes.c_void_p(buf.data_ptr())
    rows = (ctypes.c_int32 * 3)(2, 0, 8)
    bad = (ctypes.c_int32 * 3)(2, 4, 4)
    assert lib.setk_permu_align(p, None, 1, 2, 4, 8, rows, 1, p, None, None) == 0
    assert lib.setk_permu_align(p, None, 1, 2, 4, 8, bad, 1, p, None, None) == -1        # lo == hi
    assert lib.setk_permu_align(p, None, 1, 5, 4, 8, rows, 1, p, None, None) == -1       # K = 5
    assert lib.setk_permu_align(p, None, 1, 2, 4, 8, None, 0, p, None, None) == -1       # no plan
    assert lib.setk_permu_align(None, None, 1, 2, 4, 8, rows, 1, p, None, None) == -1
    assert lib.setk_cacgmm_stft(p, 1, 2, 8, 4, 2, 2, None, 0, 1, None, 0, p, None, None) == -1   # no start
    assert lib.setk_cacgmm_stft(p, 1, 1, 8, 4, 2, 2, None, 1, 1, None, 0, p, None, None) == -1   # C = 1
    assert lib.setk_cacgmm_stft(p, 1, 2, 8, 4, 2, -1, None, 1, 1, None, 0, p, None, None) == -1  # iterations
    assert lib.setk_cacgmm_stft(p, 1, 2, 8, 4, 2, 2, None, 1, 1, bad, 1, p, None, None) == -1   # plan row
    assert lib.setk_cacgmm_stft(p, 1, 2, 8, 4, 2, 2, None, 1, 1, None, 0, p, None, None) == 0


@pytest.mark.parametrize("name", ["noisy", "2spk"])
def test_doc_commands_on_the_reference_stft(emu, name):
    """The kernels fed the reference's own STFT reproduce its doc-command masks (mean <= 1e-5, max <= 5e-3)."""
    cc.check_fixture_reference_stft(emu, cc.fixture(), name)


@pytest.mark.parametrize("name", ["noisy", "nopermu", "skip"])
def test_cli(emu, emu_library_path, tmp_path, name):
    """estimate_cacgmm_masks.py: the doc enhancement command, --solve-permu false at K = 2 (K x T x F
    output), and a skipped key that draws nothing, so the next key gets the stream's first draw."""
    cc.run_cli_case(cc.fixture(), name, str(tmp_path), emu_library_path, emu)


def test_cli_init_mask_shape_error(emu_library_path, tmp_path):
    from script_runner import ROOT
    import subprocess
    import sys
    g = cc.fixture()
    scp = cc.write_fixture_inputs(g, str(tmp_path), ["noisy"])
    np.save(tmp_path / "m.npy", g["noisy/masks/noisy"][0])                  # T x F: the wrong rank
    (tmp_path / "init.scp").write_text(f"noisy {tmp_path / 'm.npy'}\n")
    code = ("import runpy, sys; sys.argv = sys.argv[1:]; from setk_b200 import _lib; "
            f"_lib.use_library({emu_library_path!r}); from setk_b200.libs import utils; "
            "utils.set_default_device('cpu'); runpy.run_path(sys.argv[0], run_name='__main__')")
    r = subprocess.run([sys.executable, "-c", code, os.path.join(ROOT, "scripts", "sptk", "estimate_cacgmm_masks.py"),
                        "--init-mask", str(tmp_path / "init.scp"), scp, str(tmp_path / "out")],
                       env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True)
    assert r.returncode != 0 and "ValueError: --init-mask must be K x T x F" in r.stderr
    assert not (tmp_path / "out" / "noisy.npy").exists()
