"""
CPU tier: the kernel sources of setk_b200/csrc compiled for the CPU execution
model (tests/emu) and driven through the same C-ABI / ctypes / plan code as the
product, checked against the oracle at small sizes.  Catches index
bookkeeping, staging, barrier-structure and argument-checking defects before a
GPU is involved.  (The sm_90a library itself is exercised by test_gpu_*.py.)
"""
import numpy as np
import pytest
import torch

import parity_cases as pc


def test_bookkeeping_bit_exact(emu):
    for fl, hop, center in [(512, 256, True), (512, 256, False), (400, 160, True),
                            (1024, 256, True), (256, 64, False)]:
        pc.check_bookkeeping(emu, fl, hop, center, [1025, 2048, 4099, 16000, 94010, 160000])


@pytest.mark.parametrize("C,N,fl,hop,center,window", [
    (1, 1500, 512, 256, True, "hann"),
    (3, 1300, 256, 128, False, "hamming"),
    (2, 2100, 1024, 256, True, "sqrthann"),
    (2, 1200, 400, 160, True, "hann"),
])
def test_stft_generic(emu, C, N, fl, hop, center, window):
    pc.check_stft(emu, np.random.default_rng(1), 1, C, N, fl, hop, center, window)


def test_non_power_of_two_n_fft(emu):
    # --round-power-of-two false --frame-len 400: n_fft = 400 through the direct-DFT route
    pc.check_non_power_of_two(emu, np.random.default_rng(12))
    with pytest.raises(Exception):
        pc.P.StftPlan(1, 401, 160, True, False, "hann", 1, 4000, emu)      # odd n_fft: librosa cannot either


def test_stft_generic_ragged(emu):
    ns = torch.tensor([1500, 900], dtype=torch.int32)
    pc.check_stft(emu, np.random.default_rng(2), 2, 2, 1500, n_samples=ns)


@pytest.mark.parametrize("C,N,hop,center,with_mn,clip,mask_ft", [
    (4, 3000, 256, True, False, False, False),     # the config-2 geometry, fused kernel
    (4, 2900, 256, False, True, False, False),
    (2, 2600, 128, True, False, True, False),
    (3, 2000, 384, True, True, False, True),
    (1, 1800, 256, True, False, False, False),
])
def test_stft_cov_fused(emu, C, N, hop, center, with_mn, clip, mask_ft):
    pc.check_stft_cov(emu, np.random.default_rng(3), 2, C, N, 512, hop, center, "hann",
                      with_mask_n=with_mn, clip=clip, mask_ft=mask_ft)


def test_stft_cov_fused_ragged(emu):
    ns = torch.tensor([3000, 1701, 2048], dtype=torch.int32)
    pc.check_stft_cov(emu, np.random.default_rng(4), 3, 4, 3000, n_samples=ns)


@pytest.mark.parametrize("B,N,hop,center,with_mn,clip,mask_ft", [
    (11, 1500, 256, True, True, True, True),     # many short utterances: CTAs own several segments
    (3, 5200, 130, True, False, False, False),   # hop % 4 != 0: every tile staged element-wise
    (2, 4100, 128, False, False, True, False),   # center=False tail feeds max|x|
    (5, 2300, 512, True, True, False, False),    # hop = n_fft (no overlap), mask_n rows
])
def test_stft_cov_ws_protocol(emu, B, N, hop, center, with_mn, clip, mask_ft):
    # the warp-specialised build (stft_cov_ws.cu): ring of Z tiles, named barriers, bin 128 rows
    pc.check_stft_cov(emu, np.random.default_rng(7), B, 4, N, 512, hop, center, "hann",
                      with_mask_n=with_mn, clip=clip, mask_ft=mask_ft)


@pytest.mark.parametrize("B,N,fl,hop,center,window,with_mn,clip", [
    (2, 3000, 512, 256, True, "hamming", True, False),   # a window other than Hann, mask_n rows
    (2, 5000, 512, 128, False, "hamming", True, False),  # hop 128 without centring
    (3, 6000, 512, 256, True, "hann", False, True),      # interior tiles between the padded edges, clip
    (1, 3000, 400, 256, True, "hann", False, False),     # 400-sample frame zero-padded to 512
])
def test_stft_cov_ws_windows(emu, B, N, fl, hop, center, window, with_mn, clip):
    # the warp-specialised build with other windows, frame lengths and lengths
    pc.check_stft_cov(emu, np.random.default_rng(11), B, 4, N, fl, hop, center, window,
                      with_mask_n=with_mn, clip=clip)


def test_stft_cov_ws_long_run(emu):
    # one long utterance: every CTA refills its 8-entry tile table (CPU build) several times
    pc.check_stft_cov(emu, np.random.default_rng(10), 1, 4, 40000)


def test_stft_cov_ws_ragged_short(emu):
    # utterances too short for one frame get an empty tile; others end mid-tile
    ns = torch.tensor([3000, 200, 1701, 513, 2999, 256, 257, 1024], dtype=torch.int32)
    pc.check_stft_cov(emu, np.random.default_rng(8), 8, 4, 3000, n_samples=ns)
    pc.check_stft_cov(emu, np.random.default_rng(9), 8, 4, 3000, 512, 256, False, "hamming",
                      n_samples=ns, with_mask_n=True)


def test_stft_cov_generic_route(emu):
    # C = 5 and n_fft = 256 have no fused instantiation: explicit STFT + covariance
    pc.check_stft_cov(emu, np.random.default_rng(5), 1, 5, 1500, 512, 256, True, "hann")
    pc.check_stft_cov(emu, np.random.default_rng(6), 1, 2, 900, 256, 64, True, "hann",
                      with_mask_n=True)


@pytest.mark.parametrize("C", [5, 6, 8, 11])
def test_many_channel_routes(emu, C):
    # C > 4 at n_fft = 512: STFT spill + streaming covariance; apply+iSTFT in
    # accumulated channel blocks of <= 4
    rng = np.random.default_rng(50 + C)
    pc.check_stft_cov(emu, rng, 2, C, 2300, 512, 256, True, "hann", with_mask_n=(C == 6),
                      clip=(C == 8))
    pc.check_apply_istft(emu, rng, 2, C, 2300, 512, 256, True, "hann", post_mask=(C == 6))


def test_many_channel_ragged_and_nocenter(emu):
    rng = np.random.default_rng(60)
    ns = torch.tensor([3000, 1701], dtype=torch.int32)
    pc.check_stft_cov(emu, rng, 2, 6, 3000, n_samples=ns)
    pc.check_apply_istft(emu, rng, 2, 6, 3000, n_samples=ns)
    pc.check_stft_cov(emu, rng, 1, 7, 2500, 512, 256, False, "hamming")
    pc.check_apply_istft(emu, rng, 1, 7, 2500, 512, 128, False, "hamming")
    # longer than the covariance kernel's cp.async ring (4 steps of 8 frames): slots are re-used
    pc.check_stft_cov(emu, rng, 1, 8, 11000, clip=True)
    pc.check_stft_cov(emu, rng, 1, 12, 9300, with_mask_n=True)


@pytest.mark.parametrize("C,hop,center", [(8, 256, True), (3, 512, False), (1, 128, True), (6, 340, True)])
def test_nfft1024_routes(emu, C, hop, center):
    # config-3 geometry: 1024-point tile STFT (even/odd half-warp jobs) into the
    # workspace, streaming covariance, w^H x + inverse FFT over the workspace
    rng = np.random.default_rng(70 + C)
    pc.check_stft_cov(emu, rng, 2, C, 4200, 1024, hop, center, "hann", with_mask_n=(C == 3),
                      clip=(C == 1))
    pc.check_apply_istft(emu, rng, 2, C, 4200, 1024, hop, center, "hann", post_mask=(C == 3))


def test_nfft1024_ragged(emu):
    rng = np.random.default_rng(75)
    ns = torch.tensor([5000, 2703], dtype=torch.int32)
    pc.check_stft_cov(emu, rng, 2, 5, 5000, 1024, 256, True, "hann", n_samples=ns)
    pc.check_apply_istft(emu, rng, 2, 5, 5000, 1024, 256, True, "hann", n_samples=ns)
    pc.check_apply_istft(emu, rng, 2, 2, 3000, 256, 64, True, "hann",
                         n_samples=torch.tensor([3000, 1501], dtype=torch.int32))   # generic route


@pytest.mark.parametrize("C,fl,K,init,alpha", [
    (4, 512, 2, False, False),        # the documented command: 2 classes, deterministic start
    (3, 1024, 3, True, True),         # given posteriors, 3 classes, prior update
    (9, 512, 2, False, False),        # C > 8: 32-bin CTAs, 5 entries per thread
])
def test_cgmm_masks(emu, C, fl, K, init, alpha):
    rng = np.random.default_rng(80 + C)
    # (C = 9 on the CPU model: 256-thread CTAs of OS threads -- one utterance, two iterations)
    B, N, iters = (1, 2800, 2) if C == 9 else (2, 4600, 3)
    pc.check_cgmm(emu, rng, B, C, N, fl, 256, K, iters, with_init=init, update_alpha=alpha,
                  n_samples=torch.tensor([4600, 3300], dtype=torch.int32) if C == 3 else None)


def test_cgmm_reference_fixtures(emu):
    for name in ("k3_alpha", "k2_init"):
        pc.check_cgmm_fixture(emu, name)


def test_cgmm_argument_errors(emu):
    from setk_b200 import plan as P
    pl = P.StftPlan(2, 512, 256, True, True, "hann", 1, 3000, emu)
    x = torch.zeros((1, 2, 3000))
    with pytest.raises(Exception):
        pl.cgmm_masks(x, 3, 2)                   # 3 classes need a start
    with pytest.raises(Exception):
        pl.cgmm_masks(x, 5, 2, init_gamma=torch.zeros((1, 5, pl.num_frames(3000), 257)))
    pl.close()
    pl = P.StftPlan(2, 256, 64, True, True, "hann", 1, 3000, emu)
    with pytest.raises(Exception):
        pl.cgmm_masks(x, 2, 2)                   # n_fft 256: no tile STFT
    pl.close()


def test_wpe(emu):
    rng = np.random.default_rng(90)
    pc.check_wpe(emu, rng, 2, 3, 2000, 256, 64, taps=4, delay=2, ctx=1, iters=2)
    pc.check_wpe(emu, rng, 1, 2, 2000, 256, 64, taps=6, delay=1, ctx=0, iters=1)
    pc.check_wpe(emu, rng, 1, 5, 3000, 256, 128, taps=3, delay=3, ctx=2, iters=2)   # NK = 15: ragged tiles
    pc.check_wpe(emu, rng, 1, 3, 3000, 256, 64, taps=4, delay=2, ctx=1, iters=2)


def test_wpe_chunked_long_utterance_path(emu, monkeypatch):
    # utterances whose bin does not fit in shared memory are walked in chunks (history +
    # context halo reloaded per chunk); forcing tiny chunks must not change a bit
    rng = np.random.default_rng(21)
    ref = pc.check_wpe(emu, rng, 1, 3, 2000, 256, 64, taps=4, delay=2, ctx=1, iters=2, return_out=True)
    for chunk in ("7", "20"):
        monkeypatch.setenv("SETK_WPE_CHUNK", chunk)
        rng = np.random.default_rng(21)
        out = pc.check_wpe(emu, rng, 1, 3, 2000, 256, 64, taps=4, delay=2, ctx=1, iters=2,
                           return_out=True)
        assert np.array_equal(out, ref)


def test_wpe_reference_fixture(emu):
    pc.check_wpe_fixture(emu, "c2_t6_ctx0")


def test_wpe_argument_errors(emu):
    from setk_b200 import plan as P
    x = torch.zeros((1, 2, 33, 20), dtype=torch.complex64)
    with pytest.raises(Exception):
        P.wpe_from_stft(x, num_iters=0)
    with pytest.raises(Exception):
        P.wpe_from_stft(torch.zeros((1, 16, 33, 20), dtype=torch.complex64), taps=10)   # NK = 160
    out, st = P.wpe_from_stft(x, taps=2, delay=1, num_iters=1)       # silence: singular normal matrix
    assert int(st[0]) != 0


def test_spatial_features(emu):
    rng = np.random.default_rng(95)
    pc.check_spatial(emu, rng, 3, 2200, 128, 64)
    pc.check_spatial(emu, rng, 2, 1500, 64, 32)


def test_spatial_argument_errors(emu):
    from setk_b200 import plan as P
    a = torch.zeros((5, 9), dtype=torch.complex64)
    with pytest.raises(ValueError):
        P.ipd(a, torch.zeros((5, 8), dtype=torch.complex64))
    with pytest.raises(ValueError):
        P.directional_feats(torch.zeros((1, 3, 9, 5), dtype=torch.complex64),
                            torch.zeros((2, 9), dtype=torch.complex128))
    with pytest.raises(ValueError):
        P.directional_feats(torch.zeros((1, 3, 9, 5), dtype=torch.complex64),
                            torch.zeros((3, 9), dtype=torch.complex128), pairs=[(0, 3)])
    with pytest.raises(ValueError):
        P.gcc_phat(a, a, np.zeros(8), np.zeros(4))
    with pytest.raises(Exception):
        P.msc(torch.zeros((1, 5, 9), dtype=torch.complex64))       # one channel: N (N - 1) = 0
    # silence: 0 / 0 like the reference (NaN everywhere, no crash)
    assert bool(torch.isnan(P.msc(torch.zeros((2, 4, 5), dtype=torch.complex64))).all())


def test_cov_generic(emu):
    pc.check_cov_generic(emu, np.random.default_rng(7), 2, 6, 9, 70)


@pytest.mark.parametrize("C", [1, 2, 4, 5, 8])
def test_weights_all_kinds(emu, C):
    pc.check_weights(emu, np.random.default_rng(10 + C), 2, 7, C)


def test_weights_c4_thread_groups(emu):
    # C = 4: eigenvector kinds on 4 threads per problem, Cholesky kinds one thread per problem
    pc.check_weights(emu, np.random.default_rng(14), 2, 7, 4)
    pc.check_weights_status(emu, C=4)


def test_weights_c64_and_status(emu):
    pc.check_weights(emu, np.random.default_rng(20), 1, 5, 4, dtype=np.complex64)
    pc.check_weights_status(emu)
    pc.check_weights_status(emu, C=6)          # the thread-group kernels of weights_coop.cu


@pytest.mark.parametrize("C,N,hop,center,pm,norm", [
    (4, 3000, 256, True, False, True),
    (4, 2500, 256, False, True, True),
    (2, 3100, 128, True, False, False),
    (3, 2000, 384, True, True, True),
])
def test_apply_istft_fused(emu, C, N, hop, center, pm, norm):
    pc.check_apply_istft(emu, np.random.default_rng(30), 2, C, N, 512, hop, center, "hann",
                         post_mask=pm, norm=norm)


def test_apply_istft_nsamps_and_ragged(emu):
    rng = np.random.default_rng(31)
    pc.check_apply_istft(emu, rng, 1, 4, 3000, n_out=3000)           # fix_length: pad
    pc.check_apply_istft(emu, rng, 1, 4, 3000, n_out=2000)           # fix_length: crop
    ns = torch.tensor([3000, 1900], dtype=torch.int32)
    pc.check_apply_istft(emu, rng, 2, 4, 3000, n_samples=ns)


def test_generic_chain(emu):
    rng = np.random.default_rng(32)
    pc.check_generic_chain(emu, rng, 1, 5, 1500, 512, 256, True, "hann")
    pc.check_generic_chain(emu, rng, 1, 2, 1000, 256, 64, False, "hamming")
    pc.check_apply_istft(emu, rng, 1, 2, 1100, 256, 128, True, "hann")   # generic apply_istft route


def test_pipeline_end_to_end_small(emu):
    from setk_b200 import synth
    x, m = synth.make_batch(1, 4, 4000, device="cpu")
    for kind in ("mvdr", "gevd", "pmwf-0"):
        err = pc.mvdr_end_to_end(emu, x.numpy(), m.numpy(), kind=kind)
        assert err <= pc.TOL_E2E, (kind, err)


def test_argument_errors(emu):
    from setk_b200 import _lib, plan as P
    with pytest.raises(_lib.SetkError):
        P.StftPlan(4, 301, 100, True, False, "hann", 1, 1000, emu)      # odd n_fft: librosa's istft cannot either
    pl = P.StftPlan(4, 512, 256, True, True, "hann", 1, 2000, emu)
    with pytest.raises(ValueError):
        pl.stft(torch.zeros(1, 3, 2000))                                # wrong channel count
    with pytest.raises(_lib.SetkError):
        pl.stft(torch.zeros(2, 4, 2000))                                # batch > max_batch
    with pytest.raises(ValueError):
        pl.stft_cov(torch.zeros(1, 4, 2000), torch.zeros(1, 3, 257))    # wrong mask shape
    with pytest.raises(ValueError):
        pl.num_frames(100)


def test_pcm_conversions(emu):
    pc.check_pcm(emu, np.random.default_rng(40))


def test_cm_masks(emu):
    pc.check_cm_masks(emu, np.random.default_rng(41))
    pc.check_cm_masks(emu, np.random.default_rng(42), B=2, T=33, F=40)
