"""
CPU tier of AuxIVA (csrc/auxiva.cuh, setk_auxiva_stft): the float64 oracle against the reference's
stored separation, the kernels' own sources on the CPU execution model (tests/emu) against the
oracle and the reference fixtures, singular utterances, the C-ABI's argument checks, and the
apply_auxiva.py command line.
"""
import numpy as np
import pytest
import torch

import auxiva_cases as ac
from oracle import auxiva_oracle as ao

G = ac.load_fixture()


@pytest.mark.parametrize("name", ac.NAMES)
def test_oracle_reproduces_reference(name):
    X = ac.fixture_stft(G[name + "/pcm16"])
    Y = ao.auxiva(X, ac.EPOCHS)[:, :, ::ac.BIN_STEP]
    want = G[name + "/Y_bins"]
    assert Y.dtype == np.complex128
    assert ac.rel_err(Y, want) <= 1e-12


@pytest.mark.parametrize("epochs", [0, 1, 3, 20])
@pytest.mark.parametrize("N", [2, 3, 4, 7, 8, 16])
def test_emu_vs_float64_oracle(emu, N, epochs):
    # 16 channels over 37 frames is too ill-conditioned for 20 epochs to keep 1e-9 in any fp64
    # summation order; more frames keep it well posed
    T = 160 if (N == 16 and epochs == 20) else 37
    ac.run_parity(emu, 2, N, 9, T, epochs, np.random.default_rng(1000 * N + epochs))


def test_emu_reference_fixtures(emu):
    ac.run_fixtures(emu)


def test_emu_zero_input_returns_input_at_zero_epochs(emu):
    from setk_b200 import plan
    X = ac.mixture(np.random.default_rng(5), 1, 3, 5, 11)
    Y, status = plan.auxiva_from_stft(torch.from_numpy(X), num_epochs=0)
    assert not status.any()
    np.testing.assert_array_equal(Y.numpy(), X.astype(np.complex128))


def test_emu_singular_bin_flags_only_its_utterance(emu):
    from setk_b200 import _lib, plan
    B, N, F, T, epochs = 3, 4, 9, 37, 3
    X = ac.mixture(np.random.default_rng(7), B, N, F, T)
    X[1, :, 4, :] = 0                                       # an all-zero bin in utterance 1
    Y, status = plan.auxiva_from_stft(torch.from_numpy(X), num_epochs=epochs)
    status, Y = status.numpy(), Y.numpy()
    assert status[1] & _lib.ST_SINGULAR
    assert status[0] == 0 and status[2] == 0
    Yo, bad = ao.auxiva_bnft(X, epochs)
    assert list(bad) == [False, True, False]
    for b in (0, 2):
        assert ac.rel_err(Y[b], Yo[b]) <= ac.TOL


def test_emu_argument_errors(emu):
    from setk_b200 import _lib
    lib = _lib.library()
    B, N, F, T = 1, 4, 5, 8
    X = np.zeros((B, 16, F, T), np.complex64)
    Y = np.zeros((B, 17, F, T), np.complex128)
    st = np.zeros(B, np.uint32)

    def call(N=N, epochs=1, x=X.ctypes.data, y=Y.ctypes.data, F=F, T=T, B=B):
        return lib.setk_auxiva_stft(x, B, N, F, T, epochs, y, st.ctypes.data, None)

    X[:] = ac.mixture(np.random.default_rng(3), B, 16, F, T)
    assert call() == 0
    assert call(N=16) == 0
    assert call(N=2, epochs=0) == 0
    assert call(N=1) == _lib.SETK_EINVAL
    assert call(N=17) == _lib.SETK_EINVAL
    assert call(epochs=-1) == _lib.SETK_EINVAL
    assert call(x=None) == _lib.SETK_EINVAL
    assert call(y=None) == _lib.SETK_EINVAL
    assert call(F=0) == _lib.SETK_EINVAL
    assert call(T=0) == _lib.SETK_EINVAL
    assert call(B=0) == _lib.SETK_EINVAL


def test_emu_apply_auxiva_matches_reference_files(tmp_path, emu_library_path):
    ac.check_cli(tmp_path, emu_library_path)


def test_emu_mirror_auxiva_signature(emu):
    """apply_auxiva.auxiva keeps the reference's N x T x F in / out and raises LinAlgError."""
    import importlib.util
    import os
    from setk_b200.libs import utils
    spec = importlib.util.spec_from_file_location("apply_auxiva", os.path.join(ac.ROOT, "scripts", "sptk",
                                                                               "apply_auxiva.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    utils.set_default_device("cpu")
    try:
        X = ac.mixture(np.random.default_rng(11), 1, 3, 7, 20)[0].transpose(0, 2, 1)      # N x T x F
        Y = mod.auxiva(X, epochs=2)
        assert isinstance(Y, np.ndarray) and Y.dtype == np.complex128 and Y.shape == X.shape
        assert ac.rel_err(Y, ao.auxiva(X, 2)) <= ac.TOL
        X[:, :, 3] = 0
        with pytest.raises(np.linalg.LinAlgError):
            mod.auxiva(X, epochs=1)
    finally:
        utils.set_default_device(None)
