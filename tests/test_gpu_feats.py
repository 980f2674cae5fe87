"""
Spectral features on the H100: the kernels of both routes against the oracle, a ragged batch larger than
the SM count, every fixture run fed from audio, run-to-run bit identity, a full-size batch and both
command lines against the reference's fixture.
"""
import numpy as np
import pytest
import torch

import feats_cases as fc
from test_feats import cli_against_fixture

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("C,fl,hop,center,window,rp2,n_mels,pw,log", [
    (1, 32, 8, True, "hann", True, 8, False, True),
    (1, 400, 160, True, "hann", False, 40, False, True),
    (2, 2048, 333, False, "hamming", True, None, True, False),
    (1, 512, 256, True, "hann", True, None, False, True),
    (5, 400, 128, False, "sqrthann", True, None, True, False),
    (4, 512, 254, True, "hann", True, 80, False, True),
    (1, 1024, 256, True, "hann", True, 64, False, True),
    (5, 1024, 512, False, "hann", True, None, False, False),
    (9, 512, 160, True, "hann", True, 40, False, False),
])
def test_kernels_vs_oracle(cuda, C, fl, hop, center, window, rp2, n_mels, pw, log):
    rng = np.random.default_rng(fl + hop + C)
    fc.check_plan(cuda, rng, C, fl, hop, center, window, rp2, (32000, 17000, 9000), n_mels, pw, log)


@pytest.mark.parametrize("fl,rp2", [(512, True), (1024, True), (400, False)])
def test_ragged_batch_beyond_sm_count(cuda, fl, rp2):
    """B = 300 with lengths at frame boundaries and the shortest accepted input: each equals it alone."""
    from setk_b200 import plan as P
    from setk_b200.libs.filters import mel
    rng = np.random.default_rng(fl)
    pl0 = P.StftPlan(1, fl, 256, True, rp2, "hann", 1, 16000, cuda)
    shortest = pl0.n_fft // 2 + 1
    lens = [int(v) for v in rng.integers(shortest, 16000, size=300)]
    lens[:4] = [shortest, 256 * 20, 256 * 20 + 1, 16000]
    N = max(lens)
    x = torch.zeros((300, 1, N), device=cuda)
    for b, n in enumerate(lens):
        x[b, 0, :n] = torch.from_numpy(rng.standard_normal(n).astype(np.float32)).to(cuda)
    pl = P.StftPlan(1, fl, 256, True, rp2, "hann", 300, N, cuda)
    pl.set_mel(mel(16000, pl.n_fft, n_mels=80, htk=True))
    ns = torch.tensor(lens, dtype=torch.int32, device=cuda)
    out = pl.spectral_feats(x, n_samples=ns, mel=True, apply_log=True)
    again = pl.spectral_feats(x, n_samples=ns, mel=True, apply_log=True)
    assert torch.equal(out, again)
    out = out.cpu().numpy()
    for b in list(range(6)) + list(rng.integers(6, 300, size=10)):
        n = lens[b]
        alone = pl.spectral_feats(x[b:b + 1, :, :n].contiguous(), mel=True, apply_log=True).cpu().numpy()[0]
        T = alone.shape[1]
        assert np.array_equal(out[b, :, :T], alone), b
        assert not out[b, :, T:].any()


def test_every_fixture_run_from_audio(cuda):
    g = fc.fixture()
    report = {}
    for name in fc.fixture_runs(g):
        _, keys, _ = fc.run_info(g, name)
        for k in keys:
            got, lin, log, pw = fc.fixture_features(cuda, g, name, k)
            ref = g[f"{name}/feats/{k}"]
            assert got.shape == ref.shape
            report[name] = fc.compare(got, lin, log, pw)
    print("fixture runs (rel-inf, max |dlog|):", report)


def test_full_size_batch(cuda):
    """256 x 10 s at 512 / 256, 80-bin log fbank, against the oracle on a sample of utterances."""
    from setk_b200 import plan as P
    from setk_b200.libs.filters import mel
    rng = np.random.default_rng(10)
    B, N = 256, 160000
    x = torch.from_numpy((rng.standard_normal((B, 1, N)) * 0.1).astype(np.float32)).to(cuda)
    pl = P.StftPlan(1, 512, 256, True, True, "hann", B, N, cuda)
    w = mel(16000, 512, n_mels=80, htk=True)
    pl.set_mel(w)
    out = pl.spectral_feats(x, mel=True, apply_log=True).cpu().numpy()
    xs = x.cpu().numpy()
    for b in (0, 77, 255):
        ref = fc.oracle_linear(xs[b], 512, 256, True, True, "hann", weights=w)
        fc.compare(out[b], ref, True)


def test_cli_against_fixture(cuda, tmp_path):
    g = fc.fixture()
    report = cli_against_fixture(g, str(tmp_path), library=None, batch_sizes=(1, 64))
    print("command lines (rel-inf, max |dlog|):", report)
