"""
GPU tier of the sound source localisation feature: setk_ssl on the H100 at full size (A = 360,
M = 8, T = 626, F = 257, B = 16) against the float64 oracle, the reference fixtures, run-to-run
bit identity, and scripts/sptk/do_ssl.py end to end.
"""
import numpy as np
import pytest
import torch

import ssl_cases as sc
from oracle import ssl_oracle as so

pytestmark = pytest.mark.gpu

B, M, F, T, A = 16, 8, 257, 626, 360
PAIRS = [(i, i + 1) for i in range(M - 1)]


def _oracle_chunked(backend, X, sv, mask, s, e, **kw):
    """The float64 oracle over direction chunks (every score depends on its own direction only)."""
    parts = [sc.oracle_window(backend, X, sv[a:a + 40], mask, s, e, **kw)[1] for a in range(0, A, 40)]
    scores = np.concatenate(parts)
    return (np.argmin(scores) if backend == "music" else np.argmax(scores)), scores


@pytest.fixture(scope="module")
def data():
    rng = np.random.default_rng(2026)
    X, sv = sc.synth(rng, B, M, F, T, A)
    mask = rng.uniform(0, 1, (B, 1, T, F)).astype(np.float32)
    mask[:, :, :, 100] = 0
    win = np.array([[(0, T), (100, 400)] for _ in range(B)], np.int32)
    win[B - 1, 0] = (0, T - 77)                                   # a ragged utterance
    return X, sv, mask, win


@pytest.mark.parametrize("backend", ["ml", "srp", "music"])
def test_fullsize_parity(cuda, data, backend):
    from setk_b200 import plan
    X, sv, mask, win = data
    kw = dict(compression=-1, eps=so.EPSILON) if backend == "ml" else {}
    if backend == "srp":
        kw["pairs"] = PAIRS
    scores, index = plan.ssl(torch.from_numpy(X).to(cuda), torch.from_numpy(sv).to(cuda), backend=backend,
                             mask=torch.from_numpy(mask).to(cuda), windows=win, **kw)
    scores, index = scores.cpu().numpy(), index.cpu().numpy()
    okw = dict(compression=-1, eps=so.EPSILON) if backend == "ml" else {}
    if backend == "srp":
        okw = dict(srp_pair=([p[0] for p in PAIRS], [p[1] for p in PAIRS]))
    for b in (0, B - 1):
        for w, (s, e) in enumerate(win[b]):
            idx_o, sc_o = _oracle_chunked(backend, X[b], sv, mask[b, 0], s, e, **okw)
            sc.check_scores(scores[b, 0, w], sc_o, index[b, 0, w], idx_o, sc.TOL_F64, f"{backend} b={b} w={w}")


def test_reference_fixtures(cuda):
    sc.run_fixtures(cuda)


@pytest.mark.parametrize("backend", ["ml", "srp", "music"])
def test_two_calls_bit_identical(cuda, data, backend):
    from setk_b200 import plan
    X, sv, mask, win = data
    args = (torch.from_numpy(X).to(cuda), torch.from_numpy(sv).to(cuda))
    kw = dict(backend=backend, mask=torch.from_numpy(mask).to(cuda), windows=win,
              pairs=PAIRS if backend == "srp" else None)
    s1, i1 = plan.ssl(*args, **kw)
    s2, i2 = plan.ssl(*args, **kw)
    assert torch.equal(s1.view(torch.int64), s2.view(torch.int64)) and torch.equal(i1, i2)


def test_do_ssl_cli(cuda, tmp_path):
    sc.check_cli(tmp_path)
    (tmp_path / "online").mkdir()
    sc.check_cli_online_mask(tmp_path / "online")
