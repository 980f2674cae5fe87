"""
GPU tier: libsetk_b200.so (sm_90a) through the C-ABI against the CPU oracle
and the golden fixtures generated from the reference's own code.
"""
import os

import numpy as np
import pytest
import torch

import parity_cases as pc
from oracle import beamformer_oracle as bo
from oracle import stft_oracle as so

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_native_library_is_loaded(cuda):
    from setk_b200 import _lib
    assert _lib.library_path().endswith("setk_b200/libsetk_b200.so")
    with open("/proc/self/maps") as f:
        assert "libsetk_b200.so" in f.read()


def test_bookkeeping_bit_exact(cuda):
    for fl, hop, center in [(512, 256, True), (512, 256, False), (400, 160, True),
                            (1024, 256, True), (256, 64, False)]:
        pc.check_bookkeeping(cuda, fl, hop, center, [1025, 2048, 4099, 16000, 94010, 160000])


@pytest.mark.parametrize("C,N,fl,hop,center,window", [
    (1, 16000, 512, 256, True, "hann"),
    (3, 9000, 256, 128, False, "hamming"),
    (8, 12000, 1024, 256, True, "sqrthann"),
    (5, 7000, 400, 160, True, "hann"),
    (2, 30000, 2048, 512, True, "blackman"),
])
def test_stft_generic(cuda, C, N, fl, hop, center, window):
    pc.check_stft(cuda, np.random.default_rng(1), 2, C, N, fl, hop, center, window)


def test_stft_generic_ragged(cuda):
    ns = torch.tensor([16000, 9000, 700], dtype=torch.int32)
    pc.check_stft(cuda, np.random.default_rng(2), 3, 2, 16000, n_samples=ns)


@pytest.mark.parametrize("C,N,hop,center,with_mn,clip,mask_ft", [
    (4, 32000, 256, True, False, False, False),
    (4, 31000, 256, False, True, False, False),
    (2, 20000, 128, True, False, True, False),
    (3, 20000, 384, True, True, False, True),
    (1, 16000, 256, True, False, False, False),
    (4, 160000, 256, True, False, True, False),    # config-2 utterance length
])
def test_stft_cov_fused(cuda, C, N, hop, center, with_mn, clip, mask_ft):
    pc.check_stft_cov(cuda, np.random.default_rng(3), 3, C, N, 512, hop, center, "hann",
                      with_mask_n=with_mn, clip=clip, mask_ft=mask_ft)


def test_stft_cov_fused_ragged(cuda):
    ns = torch.tensor([30000, 17001, 20480, 600], dtype=torch.int32)
    pc.check_stft_cov(cuda, np.random.default_rng(4), 4, 4, 30000, n_samples=ns)
    ns = torch.tensor([30000, 19000, 9000], dtype=torch.int32)
    pc.check_stft_cov(cuda, np.random.default_rng(41), 3, 4, 30000, n_samples=ns)


def test_stft_cov_generic_route(cuda):
    pc.check_stft_cov(cuda, np.random.default_rng(5), 2, 8, 16000, 1024, 256, True, "hann")   # config-3 geometry
    pc.check_stft_cov(cuda, np.random.default_rng(6), 2, 6, 9000, 512, 256, True, "hann",
                      with_mask_n=True)                                                        # config-4 channels
    pc.check_stft_cov(cuda, np.random.default_rng(7), 1, 16, 8000, 512, 256, True, "hann")
    pc.check_stft_cov(cuda, np.random.default_rng(41), 2, 8, 20000)                          # tensor-core covariance


@pytest.mark.parametrize("C", [5, 6, 8, 16])
def test_many_channel_routes(cuda, C):
    """C > 4 at n_fft = 512 (configs 4 and 5): STFT spill + streaming covariance,
    apply+iSTFT in accumulated channel blocks."""
    rng = np.random.default_rng(50 + C)
    pc.check_stft_cov(cuda, rng, 3, C, 24000, 512, 256, True, "hann", with_mask_n=(C == 6),
                      clip=(C == 8))
    pc.check_apply_istft(cuda, rng, 3, C, 24000, 512, 256, True, "hann", post_mask=(C == 6))


def test_many_channel_ragged_and_nocenter(cuda):
    rng = np.random.default_rng(60)
    ns = torch.tensor([30000, 17001, 900], dtype=torch.int32)
    pc.check_stft_cov(cuda, rng, 3, 6, 30000, n_samples=ns)
    pc.check_apply_istft(cuda, rng, 3, 6, 30000, n_samples=ns)
    pc.check_stft_cov(cuda, rng, 1, 7, 25000, 512, 256, False, "hamming")
    pc.check_apply_istft(cuda, rng, 1, 7, 25000, 512, 128, False, "hamming")


def test_cov_generic(cuda):
    pc.check_cov_generic(cuda, np.random.default_rng(7), 2, 6, 33, 300)


@pytest.mark.parametrize("C", [1, 2, 3, 4, 5, 6, 8, 16])
def test_weights_all_kinds(cuda, C):
    pc.check_weights(cuda, np.random.default_rng(10 + C), 2, 64, C)


def test_weights_c64_and_status(cuda):
    pc.check_weights(cuda, np.random.default_rng(20), 2, 64, 4, dtype=np.complex64)
    pc.check_weights(cuda, np.random.default_rng(41), 3, 257, 4)     # every kind, a full set of bins
    pc.check_weights_status(cuda)
    pc.check_weights_status(cuda, C=6)         # the thread-group kernels of weights_coop.cu
    pc.check_weights_status(cuda, C=16)


@pytest.mark.parametrize("C,N,hop,center,pm,norm", [
    (4, 32000, 256, True, False, True),
    (4, 25000, 256, False, True, True),
    (2, 31000, 128, True, False, False),
    (3, 20000, 384, True, True, True),
    (4, 160000, 256, True, False, True),
])
def test_apply_istft_fused(cuda, C, N, hop, center, pm, norm):
    pc.check_apply_istft(cuda, np.random.default_rng(30), 2, C, N, 512, hop, center, "hann",
                         post_mask=pm, norm=norm)


def test_apply_istft_nsamps_and_ragged(cuda):
    rng = np.random.default_rng(31)
    pc.check_apply_istft(cuda, rng, 1, 4, 30000, n_out=30000)
    pc.check_apply_istft(cuda, rng, 1, 4, 30000, n_out=20000)
    ns = torch.tensor([30000, 19000, 1000], dtype=torch.int32)
    pc.check_apply_istft(cuda, rng, 3, 4, 30000, n_samples=ns)


def test_non_power_of_two_n_fft(cuda):
    """--round-power-of-two false (utils.py:115, opts.py:41): n_fft = frame_len = 400 / 600."""
    pc.check_non_power_of_two(cuda, np.random.default_rng(12))
    pc.check_non_power_of_two(cuda, np.random.default_rng(13), frame_len=600, hop=200, C=5, N=9000)


def test_generic_chain(cuda):
    rng = np.random.default_rng(32)
    pc.check_generic_chain(cuda, rng, 2, 5, 15000, 512, 256, True, "hann")
    pc.check_generic_chain(cuda, rng, 1, 2, 10000, 256, 64, False, "hamming")
    pc.check_generic_chain(cuda, rng, 1, 8, 12000, 1024, 256, True, "hann")
    pc.check_apply_istft(cuda, rng, 1, 8, 12000, 1024, 256, True, "hann")


@pytest.mark.parametrize("kind,kw", [
    ("mvdr", {}), ("mvdr", {"ban": True}), ("gevd", {}), ("gevd", {"ban": True}),
    ("pmwf-0", {}), ("pmwf-1", {"pmwf_ref": 1}), ("pmwf-0", {"rank1_appro": "eig"}),
    ("pmwf-0", {"rank1_appro": "gev"}),
])
def test_pipeline_end_to_end(cuda, kind, kw):
    """north_star bound: MVDR output within 1e-4 rel-inf of the reference path."""
    from setk_b200 import synth
    x, m = synth.make_batch(3, 4, 48000, device=cuda)
    err = pc.mvdr_end_to_end(cuda, x.cpu().numpy(), m.cpu().numpy(), kind=kind, **kw)
    assert err <= pc.TOL_E2E, (kind, kw, err)


# ----------------------------------------------------------------- golden ----
def test_golden_small_cases_from_reference(cuda):
    """
    tests/golden/ref_small.npz: outputs of the reference's own forward_stft /
    compute_covar / *.weight / beamform / inverse_stft (oracle/make_golden.py).
    """
    from setk_b200 import _lib, plan as P
    g = np.load(os.path.join(GOLD, "ref_small.npz"))
    for name in ("c4_512", "c5_400", "c2_256nc", "c8_1024"):
        C, N, fl, hop, center = [int(v) for v in g[name + "/cfg"]]
        window = str(g[name + "/window"])
        mix, mask = g[name + "/mix"], g[name + "/mask"]
        pl = P.StftPlan(C, fl, hop, bool(center), True, window, 1, N, cuda)
        Rs, Rn, mx = pl.stft_cov(torch.from_numpy(mix[None]).to(cuda),
                                 torch.from_numpy(mask[None]).to(cuda))
        assert bo.rel_inf(Rs[0].cpu().numpy(), g[name + "/Rs"]) <= pc.TOL_F32
        assert bo.rel_inf(Rn[0].cpu().numpy(), g[name + "/Rn"]) <= pc.TOL_F32
        tRs = torch.from_numpy(g[name + "/Rs"][None]).to(cuda)
        tRn = torch.from_numpy(g[name + "/Rn"][None]).to(cuda)
        for kind, key in ((_lib.BF_MVDR, "w_mvdr"), (_lib.BF_GEVD, "w_gev")):
            w = P.weights(kind, tRs, tRn)[0][0].cpu().numpy()
            wa = bo.align_phase(w, g[name + "/" + key])[0]
            assert bo.rel_inf(wa, g[name + "/" + key]) <= pc.TOL_W * 100
        w = P.weights(_lib.BF_PMWF, tRs, tRn, beta=1.0, ref_channel=0)[0][0].cpu().numpy()
        assert bo.rel_inf(w, g[name + "/w_pmwf1_ref0"]) <= pc.TOL_W * 100
        # reference's MVDR weights -> our apply + iSTFT == reference's waveform
        y = pl.apply_istft(torch.from_numpy(mix[None]).to(cuda),
                           torch.from_numpy(g[name + "/w_mvdr"][None]).to(cuda),
                           norm=mx)[0].cpu().numpy()
        yr = g[name + "/y_mvdr"]
        assert y.shape == yr.shape
        assert bo.rel_inf(y, yr) <= pc.TOL_F32
        pl.close()


def test_golden_doc_vectors_pmwf_chain(cuda):
    """
    The reference's shipped example (doc/adaptive_beamformer/asset): egs.wav +
    CGMM mask -> pmwf-0 / pmwf-0-eig / pmwf-0-gev .wav.  PMWF is phase
    invariant, so the shipped PCM-16 vectors pin the whole chain: our output
    must be within 1 LSB of the float64 oracle of the same chain, and within
    3 LSB (mean <= 0.5 LSB) of the shipped files, which come from the
    reference's complex64 path and are themselves ~1e-4 relative (1-2 LSB at
    this level) from the exact answer (SURVEY.md finding 5; the reference's own
    c64 replay already differs from them: tests/golden/PINNING.json).
    """
    from setk_b200.engine import BeamformPipeline
    from setk_b200 import plan as P
    g = np.load(os.path.join(GOLD, "doc_adaptive_beamformer.npz"))
    pcm = torch.from_numpy(g["egs_pcm16"]).to(cuda)                 # (5, 94010) int16
    audio = P.pcm16_to_float(pcm)[None]
    mask = torch.from_numpy(g["mask"]).to(cuda)[None]
    for name, r1 in (("pmwf-0", ""), ("pmwf-0-eig", "eig"), ("pmwf-0-gev", "gev")):
        pipe = BeamformPipeline(5, "pmwf-0", rank1_appro=r1, max_batch=1,
                                max_samples=audio.shape[-1], device=cuda)
        wave, status = pipe.run(audio, mask)
        assert int(status[0]) == 0
        out = P.float_to_pcm16(wave)[0].cpu().numpy().astype(np.int64)
        shipped = g["shipped/" + name].astype(np.int64)
        assert out.shape == shipped.shape == (93952,)
        d = np.abs(out - shipped)
        # the shipped file is the reference's complex64 path, itself ~1e-4 rel
        # (about 1 LSB at this level) from the exact answer (SURVEY.md finding 5)
        # (so 1 LSB of ours + up to 2 LSB of the shipped file's own error)
        assert d.max() <= 3, (name, d.max())
        assert d.mean() <= 0.5, (name, float(d.mean()))
        # against the float64 oracle of the same chain: at most the odd LSB
        samps = so.float_from_pcm16(g["egs_pcm16"])
        y_o, _, _ = bo.enhance_utterance(samps, g["mask"], kind="pmwf", beta=0, rank1_appro=r1)
        d64 = np.abs(out - so.pcm16_from_float(y_o).astype(np.int64))
        # (fp32 kernels: a ~5e-7 relative error flips floor() for a few % of samples)
        assert d64.max() <= 1, (name, d64.max())
        assert np.mean(d64 > 0) <= 0.05, (name, float(np.mean(d64 > 0)))


def test_golden_doc_vectors_gevd_sign_fit(cuda):
    """
    gevd.wav is a golden vector modulo one sign per bin (scipy's hegvd chooses
    it): fit the 257 signs in the time domain (iSTFT is linear) and compare.
    """
    from setk_b200.engine import BeamformPipeline
    from setk_b200 import plan as P
    g = np.load(os.path.join(GOLD, "doc_adaptive_beamformer.npz"))
    audio = P.pcm16_to_float(torch.from_numpy(g["egs_pcm16"]).to(cuda))[None]
    mask = torch.from_numpy(g["mask"]).to(cuda)[None]
    N = audio.shape[-1]
    pipe = BeamformPipeline(5, "gevd", max_batch=1, max_samples=N, device=cuda)
    Rs, Rn, mx = pipe.covariances(audio, mask)
    w = pipe.solve(Rs, Rn)[0]
    shipped = g["shipped/gevd"].astype(np.float64) / 32768.0
    F = w.shape[1]
    stft = pipe.plan.stft(audio)
    enh = P.apply_weights(stft, w)[0]                                # (F, T)
    per_bin = torch.zeros((F, F, enh.shape[-1]), dtype=torch.complex64, device=cuda)
    idx = torch.arange(F, device=cuda)
    per_bin[idx, idx] = enh
    pl1 = P.StftPlan(1, 512, 256, True, True, "hann", F, N, cuda)
    contrib = pl1.istft(per_bin).cpu().numpy().astype(np.float64)    # (F, n_out)
    signs = np.sign(contrib @ shipped)
    signs[signs == 0] = 1
    y = (signs[:, None] * contrib).sum(axis=0)
    y = y * float(mx[0]) / (np.max(np.abs(y)) + so.EPSILON)
    out = so.pcm16_from_float(y).astype(np.int64)
    d = np.abs(out - g["shipped/gevd"].astype(np.int64))
    assert d.max() <= 2, d.max()
    assert np.mean(d > 0) <= 0.05


def test_pcm_conversions(cuda):
    pc.check_pcm(cuda, np.random.default_rng(40))


def test_cm_masks(cuda):
    """Kaldi compressed-matrix masks expanded on the device (kaldi_io.py:248-281): bit-exact."""
    pc.check_cm_masks(cuda, np.random.default_rng(41))
    pc.check_cm_masks(cuda, np.random.default_rng(42), B=5, T=626, F=257)


@pytest.mark.parametrize("name", ["cfg3", "cfg4"])
def test_config_fixtures_from_reference(cuda, name):
    """configs 3 (reference CGMM mask -> GEV) and 4 (reference WPE -> MVDR)."""
    pc.check_config_fixture(cuda, name)


@pytest.mark.parametrize("C,fl,K,init,alpha,ragged", [
    (4, 512, 2, False, False, False),
    (5, 512, 2, True, False, True),
    (8, 1024, 2, False, False, False),     # config-3 geometry
    (3, 1024, 3, True, True, True),
    (6, 512, 4, True, True, False),
    (12, 512, 2, False, False, False),     # C > 8 kernels
    (16, 512, 3, True, False, False),
])
def test_cgmm_masks(cuda, C, fl, K, init, alpha, ragged):
    rng = np.random.default_rng(300 + C)
    ns = torch.tensor([16000, 9100, 12345], dtype=torch.int32) if ragged else None
    pc.check_cgmm(cuda, rng, 3, C, 16000, fl, 256, K, 8, with_init=init, update_alpha=alpha,
                  n_samples=ns)


def test_cgmm_reference_fixtures(cuda):
    """given posteriors / 3 classes / prior update, run by the reference (ref_cgmm.npz)"""
    for name in ("k3_alpha", "k2_init"):
        pc.check_cgmm_fixture(cuda, name)


@pytest.mark.parametrize("which", ["doc", "cfg3"])
def test_cgmm_documented_command_from_audio(cuda, which):
    """
    estimate_cgmm_masks.py --num-iters 20 from audio vs the reference's masks.
    This path's STFT is float32 arithmetic (rel. 3e-7) where the reference's is
    float64 rounded to complex64, and the reference's algorithm is ill-conditioned
    wherever an eigenvalue of R_k sits at its 1.19e-7 floor: feeding the oracle a
    float32 scipy FFT instead of the float64 one moves its doc-example masks by
    8e-6 on average, 6e-3 in the worst cell and > 1e-3 in 0.24 % of the cells --
    the same order as the bounds asserted here.
    """
    mean, worst, frac = pc.check_cgmm_documented(cuda, which)
    print(f"cgmm {which}: mean {mean:.3g} max {worst:.3g} frac>1e-3 {frac:.3g}")
    assert mean <= 1e-4 and frac <= 1e-2 and worst <= 0.1


@pytest.mark.parametrize("C,fl,hop,taps,delay,ctx,iters,N", [
    (6, 512, 256, 10, 3, 1, 3, 48000),      # config-4 geometry: NK = 60
    (8, 512, 128, 10, 3, 1, 2, 24000),      # NK = 80
    (6, 512, 128, 10, 3, 1, 2, 16000),
    (2, 1024, 256, 12, 2, 0, 1, 30000),
    (5, 512, 128, 3, 3, 2, 3, 16000),       # NK = 15: ragged tiles
    (1, 512, 128, 10, 3, 1, 3, 16000),
])
def test_wpe(cuda, C, fl, hop, taps, delay, ctx, iters, N):
    pc.check_wpe(cuda, np.random.default_rng(400 + C), 2, C, N, fl, hop, taps, delay, ctx, iters)


def test_wpe_reference_fixtures(cuda):
    """libs/wpe.py wpe() run by the reference (tests/golden/ref_wpe.npz)"""
    for name in ("c3_t4", "c4_t10", "c2_t6_ctx0"):
        pc.check_wpe_fixture(cuda, name)


@pytest.mark.gpu
@pytest.mark.parametrize("C,N,fl,hop", [(4, 20000, 512, 256), (2, 9000, 1024, 256), (7, 6000, 256, 64)])
def test_spatial_features(cuda, C, N, fl, hop):
    """ipd / directional_feats / gcc_phat / srp / msc kernels vs oracle/spatial_oracle.py"""
    pc.check_spatial(cuda, np.random.default_rng(500 + C), C, N, fl, hop)


@pytest.mark.gpu
def test_spatial_reference_fixtures(cuda):
    """libs/spatial.py run by the reference (tests/golden/ref_spatial.npz)"""
    for name in ("c4_512", "c3_256", "c2_1024"):
        pc.check_spatial_fixture(cuda, name)


@pytest.mark.gpu
def test_spatial_libs_mirror_numpy(cuda):
    """setk_b200.libs.spatial: the reference's names and axes, numpy in -> numpy out"""
    from oracle import spatial_oracle as sp
    from setk_b200.libs import spatial as gs
    rng = np.random.default_rng(77)
    S = (rng.standard_normal((3, 40, 129)) + 1j * rng.standard_normal((3, 40, 129))).astype(np.complex64)
    d = [0.0, 0.05, 0.1]
    kw = dict(num_bins=129, num_doa=19)
    got = gs.srp_phat_linear(S, d, **kw)
    ref = sp.srp_phat_linear(S, d, **kw)
    assert isinstance(got, np.ndarray) and got.dtype == np.float64 and got.shape == ref.shape
    assert np.max(np.abs(got - ref)) <= 5e-6 * np.max(np.abs(ref))
    assert np.max(np.abs(gs.ipd(S[0], S[1], cos=True, sin=True) - sp.ipd(S[0], S[1], cos=True, sin=True))) <= 5e-6
    assert np.max(np.abs(gs.msc(S) - sp.msc(S))) <= 1e-9
    obs = np.ascontiguousarray(np.transpose(S, (0, 2, 1)))
    sv = np.exp(1j * rng.uniform(0, 6.28, size=(3, 129)))
    assert np.max(np.abs(gs.directional_feats(obs, sv) - sp.directional_feats(obs, sv))) <= 5e-6
    assert np.array_equal(gs.linear_tdoa_grid(0.1, **kw), np.exp(-1j * np.outer(*sp.tdoa_grid(0.1, **kw))))
    with pytest.raises(ValueError):
        gs.srp_phat_linear(S, np.array(d))


@pytest.mark.gpu
def test_geometry_based_beamformers(cuda):
    """DS / SD / fixed beamformers (host weights, setk_apply on the observations) vs ref_fixed_bf.npz"""
    pc.check_fixed_beamformers(cuda)


@pytest.mark.gpu
def test_facted_wpd_reference_fixtures(cuda):
    """libs/wpe.py facted_wpd() run by the reference (tests/golden/ref_wpd.npz)"""
    from setk_b200.libs import utils
    utils.set_default_device(cuda)
    try:
        for name in ("c3", "c4"):
            pc.check_wpd_fixture(cuda, name)
    finally:
        utils.set_default_device(None)
