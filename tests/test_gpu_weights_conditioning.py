"""
GPU tier: every route of the per-bin fp64 weight solve (weights.cu, weights_coop.cu) and the
stand-alone BAN / rank-1 kernels (weights_post.cu) on the device, against the 40-digit reference
of solve_cases.py, across conditioning, rank and batch composition.  Run with -rP to see the
worst err / bound per route and dtype.
"""
import numpy as np
import pytest
import torch

import solve_cases as sc
from setk_b200 import _lib
from setk_b200 import plan as P

pytestmark = pytest.mark.gpu

CS = (1, 2, 3, 4, 5, 8, 12, 16)
DTYPES = (np.complex128, np.complex64)


@pytest.fixture(scope="module", autouse=True)
def worst_ratios():
    """Collect this module's worst err / bound per route; -rP shows them after its last test."""
    sc.WORST.clear()
    yield
    print("\nweights vs the 40-digit reference (device):\n" + sc.report())


@pytest.mark.parametrize("dtype", DTYPES, ids=("c128", "c64"))
@pytest.mark.parametrize("C", CS)
def test_sweep(cuda, C, dtype):
    # every kind x complex128 / complex64 outputs; PMWF (12 variants) at the smaller C, where the
    # reference's C column solves stay cheap
    sc.check_sweep(cuda, C, 2 if C >= 12 else 3, sc.SWEEP_FAMILIES, dtype, pmwf=C <= 8)


@pytest.mark.parametrize("C", (12, 16))
def test_sweep_pmwf_large_c(cuda, C):
    sc.check_sweep(cuda, C, 1, [("cond", 1e4), ("cond", 1e12), ("gap", 1e-7), ("pgap", 1e-7)],
                   np.complex128, kinds=[], ban=False)


@pytest.mark.parametrize("dtype", DTYPES, ids=("c128", "c64"))
@pytest.mark.parametrize("C", CS)
def test_ban_rank1(cuda, C, dtype):
    fams = [("cond", 1e1), ("cond", 1e8), ("cond", 1e12), ("gap", 1e-7), ("pgap", 1e-7), ("rank1", None),
            ("scale", -40), ("scale", 40)]
    sc.check_post(cuda, C, 2, fams, dtype)


@pytest.mark.parametrize("C", (2, 3, 4, 5, 8, 12, 16))
def test_status_contract(cuda, C):
    sc.check_dead_channel(cuda, C)
    sc.check_dead_channel(cuda, C, dead=0, seed=12)
    sc.check_ladder_depth(cuda, C)
    sc.check_rank_deficient(cuda, C)
    sc.check_silent(cuda, C)


# B * F fills several CTAs of the device's launches (C = 4: 32 groups of 4 per 128-thread CTA;
# C = 5..8: 16 groups of 8; C = 9..16: 4 groups of 16 per 64-thread CTA) and leaves a partial one.
@pytest.mark.parametrize("C,B,F", [(4, 3, 37), (5, 3, 23), (8, 3, 23), (12, 3, 7), (16, 3, 7)])
def test_batch_invariance(cuda, C, B, F):
    kinds = [("mvdr", False), ("mvdr", True), ("mpdr", False), ("pevd", False)]
    if C > 4:
        kinds += [("gevd", False), ("gevd", True), ("pevd_rn", False)]
    sc.check_invariance(cuda, C, B, F, kinds)
    sc.check_invariance(cuda, C, B, F, [("mvdr", True)] + ([("gevd", True)] if C > 4 else []), seed=9,
                        dtype=np.complex64, out=torch.complex64)


@pytest.mark.parametrize("C", CS)
def test_exact_scaling(cuda, C):
    sc.check_scaling(cuda, C)
    if C > 1:
        sc.check_eps_floor(cuda, C)


def test_fullsize_config2(cuda, B=256):
    """Config 2's shape (B = 256, F = 257, C = 4): covariances from stft_cov on synthetic audio with
    near-binary masks, so bins with cond(Rn) far above 1e5 appear.  A sample of bins, the worst
    conditioned among them, against the reference."""
    from setk_b200 import synth
    C, N = 4, 16000
    audio, irm = synth.make_batch(B, C, N, device=cuda)
    mask = torch.sigmoid(80.0 * (irm - 0.3))      # near-binary, generous to speech: few noise frames
    pl = P.StftPlan(C, 512, 256, True, True, "hann", B, N, cuda)
    Rs, Rn, _ = pl.stft_cov(audio, mask, None, want_maxabs=False)
    pl.close()
    assert Rs.shape == (B, 257, C, C)
    wm, stm, _ = P.weights(_lib.BF_MVDR, Rs, Rn, out_dtype=torch.complex128)
    wg, stg, _ = P.weights(_lib.BF_GEVD, Rs, Rn, out_dtype=torch.complex128)
    Rs64 = Rs.cpu().numpy().astype(np.complex128)
    Rn64 = Rn.cpu().numpy().astype(np.complex128)
    # a bin whose noise mask rounds to 0 in every frame has Rn = 0: the reference's LinAlgError,
    # ST_SINGULAR (MVDR) / ST_NOT_PD (GEVD) for that utterance; every other utterance is clean
    zero = ~Rn64.reshape(B, -1, C * C).any(axis=-1)
    stm, stg = stm.cpu().numpy(), stg.cpu().numpy()
    for b in range(B):
        assert (stm[b] & _lib.ST_ERROR_MASK) == (_lib.ST_SINGULAR | _lib.ST_NONFINITE if zero[b].any() else 0)
        assert (stg[b] & _lib.ST_ERROR_MASK) == (_lib.ST_NOT_PD if zero[b].any() else 0)
    wm, wg = wm.cpu().numpy(), wg.cpu().numpy()
    ev = np.linalg.eigvalsh(Rn64)
    cond = np.where(ev[..., 0] > 0, ev[..., -1] / np.maximum(ev[..., 0], 1e-300), np.inf)
    cond[zero] = 0.0
    print(f"\nconfig-2 covariances: {np.sum(cond > 1e5)} of {cond.size} bins with cond(Rn) > 1e5, "
          f"largest {np.max(cond):.3e}, {zero.sum()} with Rn = 0")
    assert np.sum(cond > 1e5) >= 20
    order = np.argsort(cond, axis=None)
    rng = np.random.default_rng(0)
    pick = list(order[-12:]) + list(rng.choice(order[zero.sum():-12], 24, replace=False))
    for i in pick:
        b, f = np.unravel_index(i, cond.shape)
        r = sc.BinRef(Rs64[b, f], Rn64[b, f])
        ref, c, al = r.mvdr()
        sc.check("mvdr config-2 fullsize c64->c128", C, wm[b, f], ref, c, False, align=al,
                 what=f"utt {b} bin {f}")
        if cond[b, f] < 1e12:     # beyond, whether the unloaded Cholesky passes is a matter of rounding
            ref, c, al = r.gevd()
            sc.check("gevd config-2 fullsize c64->c128", C, wg[b, f], ref, c, False, align=al,
                     what=f"utt {b} bin {f}")
