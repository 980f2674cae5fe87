"""
CPU tier of noise suppression (csrc/ns.cu, setk_ns_imcra): the float64 oracle against the
reference's stored gains, the kernel's own source on the CPU execution model (tests/emu) against
the oracle and the reference fixtures, ragged batches, the C-ABI's argument checks, the iMCRA
mirror and the apply_ns.py command line.
"""
import ctypes

import numpy as np
import pytest
import torch

import ns_cases as nc
from oracle import ns_oracle as no
from script_runner import run_script

G = nc.load_fixture()

CONFIGS = {
    "default": {},
    "case_b": nc.CASE_B_CONF,                          # U > V, w_mcra = 2, Hamming, other constants
    "u20_v7": dict(U=20, V=7),                         # U not a multiple of V
    "u8_v4": dict(U=8, V=4),                           # U a multiple of V
    "u3_v1": dict(U=3, V=1),                           # a sub-window per frame
    "w0": dict(w_mcra=0),                              # no smoothing across bins
}


def test_oracle_reproduces_reference_clip():
    X = nc.fixture_stft(G["egs/pcm16"])
    g = no.iMCRA().run(X)
    assert g.dtype == np.float64 and g.shape == X.shape
    assert np.max(np.abs(g[::nc.FRAME_STEP] - G["egs/gain_frames"])) <= 1e-6


@pytest.mark.parametrize("name", ["a", "b"])
def test_oracle_reproduces_reference_cases(name):
    conf = nc.CASE_B_CONF if name == "b" else {}
    g = no.iMCRA(**conf).run(G[name + "/stft"])
    assert nc.gain_err(g, G[name + "/gain"]) <= nc.TOL_REF
    assert np.all(np.isfinite(g))


def test_oracle_e1_at_zero():
    assert no.expint(0.0) == no.E1_AT_ZERO
    assert abs(no.expint(1e-30) - 68.51) < 0.01


@pytest.mark.parametrize("T", [1, 15, 16, 37, 200])
@pytest.mark.parametrize("F", [9, 33, 257, 513])
def test_emu_vs_float64_oracle(emu, F, T):
    nc.run_parity(emu, 2, F, T, {}, np.random.default_rng(100 * F + T))


@pytest.mark.parametrize("conf", list(CONFIGS), ids=list(CONFIGS))
@pytest.mark.parametrize("F,T", [(9, 37), (33, 200), (257, 61)])
def test_emu_configurations(emu, F, T, conf):
    nc.run_parity(emu, 1, F, T, CONFIGS[conf], np.random.default_rng(7 * F + T))


def test_emu_reference_cases(emu):
    nc.run_cases(emu)


def test_emu_reference_clip(emu):
    nc.run_clip(emu)


def test_emu_ragged_batch_matches_each_utterance_alone(emu):
    from setk_b200 import plan
    B, F, T = 3, 33, 37
    n_frames = [37, 20, 1]
    X = torch.from_numpy(nc.noisy_stft(np.random.default_rng(3), B, F, T))
    g, e = plan.ns_from_stft(X, n_frames=n_frames, config=nc.CASE_B_CONF)
    for b, n in enumerate(n_frames):
        g1, e1 = plan.ns_from_stft(X[b:b + 1, :, :n].contiguous(), config=nc.CASE_B_CONF)
        assert torch.equal(g[b, :n], g1[0]) and torch.equal(e[b, :, :n], e1[0])
        assert not g[b, n:].any() and not e[b, :, n:].any()
    nc.run_parity(emu, B, F, T, nc.CASE_B_CONF, np.random.default_rng(3), n_frames=n_frames)


def test_emu_outputs_alone_match_both(emu):
    from setk_b200 import plan
    X = torch.from_numpy(nc.noisy_stft(np.random.default_rng(4), 2, 33, 40))
    g, e = plan.ns_from_stft(X)
    g1, none1 = plan.ns_from_stft(X, enh=False)
    none2, e2 = plan.ns_from_stft(X, gain=False)
    assert none1 is None and none2 is None
    assert torch.equal(g, g1) and torch.equal(e, e2)


def test_emu_argument_errors(emu):
    from setk_b200 import _lib, plan
    lib = _lib.library()
    B, F, T = 1, 9, 8
    X = nc.noisy_stft(np.random.default_rng(5), B, F, T)
    g = np.zeros((B, T, F))
    e = np.zeros((B, F, T), np.complex64)

    def call(conf=None, x=X.ctypes.data, gp=g.ctypes.data, ep=e.ctypes.data, B=B, F=F, T=T, null_cfg=False,
             null_window=False):
        cfg, window = plan.imcra_config(conf)
        if null_window:
            cfg.window_host = None
        return lib.setk_ns_imcra(None if null_cfg else ctypes.byref(cfg), x, None, B, F, T, gp, ep, None)

    assert call() == 0
    assert call(dict(w_mcra=4)) == 0                               # F = 9 = 2 * 4 + 1 taps
    assert call(dict(U=64, V=1)) == 0
    assert call(null_cfg=True) == _lib.SETK_EINVAL
    assert call(null_window=True) == _lib.SETK_EINVAL
    assert call(x=None) == _lib.SETK_EINVAL
    assert call(gp=None, ep=None) == _lib.SETK_EINVAL
    assert call(gp=None) == 0 and call(ep=None) == 0
    assert call(B=0) == _lib.SETK_EINVAL
    assert call(F=0) == _lib.SETK_EINVAL
    assert call(T=0) == _lib.SETK_EINVAL
    assert call(F=_lib.NS_MAX_BINS + 1) == _lib.SETK_EINVAL
    assert call(dict(w_mcra=5)) == _lib.SETK_EINVAL                # F = 9 < 11 taps
    cfg, window = plan.imcra_config(dict(w_mcra=8))
    cfg.w_mcra = 9
    assert lib.setk_ns_imcra(ctypes.byref(cfg), X.ctypes.data, None, B, F, T, g.ctypes.data, None, None) \
        == _lib.SETK_EINVAL                                        # w_mcra outside [0, 8]
    cfg.w_mcra = -1
    assert lib.setk_ns_imcra(ctypes.byref(cfg), X.ctypes.data, None, B, F, T, g.ctypes.data, None, None) \
        == _lib.SETK_EINVAL
    assert call(dict(V=0)) == _lib.SETK_EINVAL
    assert call(dict(U=0)) == _lib.SETK_EINVAL
    assert call(dict(U=65)) == _lib.SETK_EINVAL
    with pytest.raises(ValueError):
        plan.imcra_config(dict(w_mcra=9))
    with pytest.raises(TypeError):
        plan.imcra_config(dict(delta=5))


def test_emu_mirror_imcra_run(emu):
    """libs.ns.iMCRA().run keeps the reference's T x F complex in, T x F float64 out."""
    from setk_b200.libs import utils
    from setk_b200.libs.ns import iMCRA
    utils.set_default_device("cpu")
    try:
        S = G["b/stft"]
        g = iMCRA(**nc.CASE_B_CONF).run(S)
        assert isinstance(g, np.ndarray) and g.dtype == np.float64 and g.shape == S.shape
        assert nc.gain_err(g, no.iMCRA(**nc.CASE_B_CONF).run(S)) <= nc.TOL_GAIN
    finally:
        utils.set_default_device(None)


def test_emu_apply_ns_wave_matches_reference_file(tmp_path, emu_library_path):
    nc.check_cli(tmp_path, emu_library_path)


def test_emu_apply_ns_gain_and_conf(tmp_path, emu_library_path):
    import yaml
    nc.write_cli_inputs(tmp_path)
    conf = dict(nc.CASE_B_CONF)
    (tmp_path / "ns.yaml").write_text(yaml.safe_dump(conf))
    out = tmp_path / "gain"
    run_script("apply_ns.py", [str(tmp_path / "wav.scp"), str(out), "--output", "gain", "--conf",
                               str(tmp_path / "ns.yaml")], emu_library_path)
    assert not list(out.glob("stereo.*"))
    g = np.load(out / "egs.npy")
    from oracle import stft_oracle
    from setk_b200.libs import utils
    utils.set_default_device("cpu")
    try:                                   # the oracle on the STFT the library computed
        X = utils.forward_stft(stft_oracle.float_from_pcm16(G["egs/pcm16"]), transpose=True, **nc.STFT_KW)
    finally:
        utils.set_default_device(None)
    assert g.dtype == np.float64 and g.shape == X.shape
    assert nc.gain_err(g, no.iMCRA(**conf).run(X)) <= nc.TOL_GAIN


def test_apply_ns_rejects_other_sample_rates(tmp_path, emu_library_path):
    nc.write_cli_inputs(tmp_path, with_multichannel=False)
    with pytest.raises(AssertionError, match="ValueError: Now only support audio in 16kHz"):
        run_script("apply_ns.py", [str(tmp_path / "wav.scp"), str(tmp_path / "out"), "--sr", "8000"],
                   emu_library_path)
