"""
CPU tier of the sound source localisation feature (csrc/ssl.cuh, setk_ssl): the oracle against the
reference's stored results, the kernels' own sources on the CPU execution model (tests/emu) against
the float64 oracle and the reference fixtures, the C-ABI's argument checks, and the do_ssl.py /
compute_steer_vector.py command lines.
"""
import ctypes
import json
import os

import numpy as np
import pytest

import ssl_cases as sc
from oracle import ssl_oracle as so

G = sc.load_fixture()


@pytest.mark.parametrize("name", ["lin4", "circ7", "lin2"])
def test_oracle_reproduces_reference(name):
    """Reference dtype flow: every index equal, every score within 1e-12 of max|score|."""
    S, sv = G[name + "/stft"], G[name + "/sv"]
    pairs = (list(G[name + "/pairs"][:, 0]), list(G[name + "/pairs"][:, 1]))
    eps = so.EPSILON
    calls = {
        "ml": lambda: so.ml_ssl(S, sv, compression=-1, eps=eps),
        "ml_mask": lambda: so.ml_ssl(S, sv, compression=-1, eps=eps, mask=G[name + "/mask"]),
        "ml_norm": lambda: so.ml_ssl(S, sv, norm=True, mask=G[name + "/mask"]),
        "ml_mask3": lambda: so.ml_ssl(S, sv, compression=-1, eps=eps, mask=G[name + "/mask3"]),
        "ml_pow": lambda: so.ml_ssl(S, sv, compression=0.5, mask=G[name + "/mask"]),
        "srp": lambda: so.srp_ssl(S, sv, srp_pair=pairs),
        "srp_mask": lambda: so.srp_ssl(S, sv, srp_pair=pairs, mask=G[name + "/mask"]),
        "music": lambda: so.music_ssl(S, sv),
        "music_mask": lambda: so.music_ssl(S, sv, mask=G[name + "/mask_zero_bin"]),
    }
    for run, fn in calls.items():
        idx, scores = fn()
        want = G[f"{name}/{run}/scores"]
        np.testing.assert_array_equal(idx, G[f"{name}/{run}/index"], err_msg=run)
        err = np.max(np.abs(scores - want)) / np.max(np.abs(want))
        assert err <= 1e-12, f"{run}: {err:.3e}"


def test_fixture_source_direction_is_clear():
    pin = json.load(open(os.path.join(sc.ROOT, "tests", "golden", "PINNING_ssl.json")))
    for name in ("lin4", "circ7", "lin2"):
        assert abs(pin[f"{name}/ml_index"] - pin[f"{name}/true_doa_index"]) <= 1


ML_CASES = [  # M, norm, compression, mask
    (2, False, -1.0, None), (4, True, -1.0, "2d"), (4, False, 0.5, "3d"), (6, True, 0.5, None),
    (8, False, 0.0, "2d"), (16, False, -1.0, "3d"),
]


@pytest.mark.parametrize("M,norm,compression,mask", ML_CASES)
def test_emu_ml_vs_float64_oracle(emu, M, norm, compression, mask):
    rng = np.random.default_rng(100 + M)
    sc.run_parity(emu, "ml", 2, M, 9, 37, 11, mask, rng, compression=compression, eps=so.EPSILON,
                  normalize=norm)


@pytest.mark.parametrize("M,mask", [(2, None), (4, "2d"), (7, "2d"), (16, None)])
def test_emu_srp_vs_float64_oracle(emu, M, mask):
    rng = np.random.default_rng(200 + M)
    pairs = [(i, (i + 1) % M) for i in range(M - 1)] + ([(M - 1, 0)] if M > 2 else [])
    sc.run_parity(emu, "srp", 2, M, 9, 37, 13, mask, rng, pairs=pairs)


@pytest.mark.parametrize("M,mask", [(2, None), (3, "zero_bin"), (5, "2d"), (8, "zero_bin"), (16, None)])
def test_emu_music_vs_float64_oracle(emu, M, mask):
    rng = np.random.default_rng(300 + M)
    sc.run_parity(emu, "music", 2, M, 9, 37, 10, mask, rng)


def test_emu_reference_fixtures(emu):
    sc.run_fixtures(emu)


def test_emu_mirror_api(emu):
    """libs.ssl keeps the reference's signatures, return types and errors."""
    from setk_b200.libs import ssl as L
    from setk_b200.libs import utils
    utils.set_default_device("cpu")
    try:
        S, sv = G["lin2/stft"], G["lin2/sv"]
        idx = L.ml_ssl(S, sv, compression=-1, eps=so.EPSILON)
        assert isinstance(idx, np.integer) and idx == G["lin2/ml/index"]
        idx3, scores = L.ml_ssl(S, sv, compression=-1, eps=so.EPSILON, mask=G["lin2/mask3"], return_scores=True)
        assert idx3.shape == (2,) and scores.shape == (2, sv.shape[0]) and isinstance(scores, np.ndarray)
        assert L.music_ssl(S, sv, mask=G["lin2/mask_zero_bin"]) == G["lin2/music_mask/index"]
        assert L.srp_ssl(S, sv, srp_pair=([0], [1])) == G["lin2/srp/index"]
        with pytest.raises(ValueError):
            L.srp_ssl(S, sv)
    finally:
        utils.set_default_device(None)


def test_emu_argument_errors(emu):
    from setk_b200 import _lib
    lib = _lib.library()
    B, M, F, T, A = 1, 4, 5, 8, 3
    X = np.zeros((B, M, F, T), np.complex64)
    sv = np.ones((A, M, F), np.complex128)
    mask = np.ones((B, 2, T, F), np.float32)
    scores = np.zeros((B, 2, 2, A))
    index = np.zeros((B, 2, 2), np.int32)

    def call(backend=0, M=M, A=A, steer_F=F, mask_p=None, N=1, win=((0, T),), pairs=((0, 1),)):
        w = np.ascontiguousarray(np.array(win, np.int32).reshape(B, -1, 2))
        p = np.ascontiguousarray(np.array(pairs, np.int32).reshape(-1, 2))
        return lib.setk_ssl(backend, X.ctypes.data, B, M, F, T, sv.ctypes.data, A, steer_F, mask_p, N,
                            w.ctypes.data, w.shape[1], p.ctypes.data, p.shape[0], -1.0, 1e-8, 0,
                            scores.ctypes.data, index.ctypes.data, None)

    m = mask.ctypes.data
    assert call() == 0
    assert call(backend=1) == 0
    assert call(backend=2) == 0
    assert call(backend=0, mask_p=m, N=2) == 0
    assert call(backend=3) == _lib.SETK_EINVAL
    assert call(backend=1, mask_p=m, N=2) == _lib.SETK_EINVAL
    assert call(backend=2, mask_p=m, N=2) == _lib.SETK_EINVAL
    assert call(backend=1, pairs=((0, 4),)) == _lib.SETK_EINVAL
    assert call(backend=1, pairs=((-1, 0),)) == _lib.SETK_EINVAL
    assert call(A=0) == _lib.SETK_EINVAL
    assert call(win=((0, T + 1),)) == _lib.SETK_EINVAL
    assert call(win=((3, 3),)) == _lib.SETK_EINVAL
    assert call(win=((-1, 2),)) == _lib.SETK_EINVAL
    assert call(M=17) == _lib.SETK_EINVAL
    assert call(N=2) == _lib.SETK_EINVAL                      # two masks announced, none given
    assert call(steer_F=F + 1) == _lib.SETK_ESHAPE


def test_emu_do_ssl_matches_reference_output(tmp_path, emu_library_path):
    sc.check_cli(tmp_path, emu_library_path)


def test_emu_do_ssl_online_mask_slices_time(tmp_path, emu_library_path):
    sc.check_cli_online_mask(tmp_path, emu_library_path)


def test_windows_of_online_mode():
    from setk_b200.cli_tools import ssl_windows
    assert ssl_windows(10, -1, 125) == [(0, 10)]
    assert ssl_windows(10, 4, 0) == [(0, 10)]
    assert ssl_windows(10, 4, 3) == [(0, 4), (1, 8), (5, 10)]
    assert ssl_windows(10, 4, 3) == so.online_windows(10, 4, 3)


@pytest.mark.parametrize("name", ["linear", "circular"])
def test_compute_steer_vector_matches_reference(tmp_path, name):
    from setk_b200.cli_tools import steer_vector_main
    flags = json.loads(str(G[f"steer/{name}/flags"]))
    argv = [str(tmp_path / "sv.npy"), "--num-bins", "33", "--sr", "16000", "--speed", "343"]
    for k, v in flags.items():
        if k == "linear_topo":
            v = ",".join(str(x) for x in v)
        argv += ["--" + k.replace("_", "-"), str(v)]
    steer_vector_main(argv)
    got = np.load(tmp_path / "sv.npy")
    want = G[f"steer/{name}"]
    assert got.dtype == np.complex128 and got.shape == want.shape
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-15)
