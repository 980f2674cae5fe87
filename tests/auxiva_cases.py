"""
Shared cases of the AuxIVA tests (tests/test_auxiva.py on the CPU execution model,
tests/test_gpu_auxiva.py on the device): setk_auxiva_stft through setk_b200.plan.auxiva_from_stft
against the float64 oracle (oracle/auxiva_oracle.py) and the reference fixtures
(tests/golden/ref_auxiva.npz), and scripts/sptk/apply_auxiva.py against the reference's files.
"""
import os

import numpy as np
import torch

from script_runner import run_script

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_auxiva.npz")

from oracle import auxiva_oracle as ao  # noqa: E402
from oracle import stft_oracle  # noqa: E402

NAMES = ("egs", "spk7", "mix2")
EPOCHS = 20
BIN_STEP = 32
STFT_KW = dict(frame_len=512, frame_hop=256, window="hann", center=True, round_power_of_two=True)
# Y against the float64 oracle, relative to max |Y|
TOL = 1e-9


def load_fixture():
    return dict(np.load(GOLD))


def fixture_stft(pcm):
    """N x T x F complex64 STFT of PCM-16 audio, as the reference's SpectrogramReader computes it."""
    return stft_oracle.multichannel_stft(stft_oracle.float_from_pcm16(pcm), transpose=True,
                                         out_dtype=np.complex64, **STFT_KW)


def mixture(rng, B, N, F, T):
    """B x N x F x T complex64: N super-Gaussian sources through a random N x N mixing per bin."""
    S = (rng.standard_normal((B, N, F, T)) + 1j * rng.standard_normal((B, N, F, T))) \
        * (0.2 + rng.gamma(1.0, 1.0, (B, N, 1, T)))
    A = rng.standard_normal((B, F, N, N)) + 1j * rng.standard_normal((B, F, N, N))
    return np.einsum("bfij,bjft->bift", A, S).astype(np.complex64)


def rel_err(got, want):
    return float(np.max(np.abs(got - want)) / np.max(np.abs(want)))


def run_parity(device, B, N, F, T, epochs, rng, check=None):
    """plan.auxiva_from_stft vs the float64 oracle on utterances `check` (default: all)."""
    from setk_b200 import plan
    X = mixture(rng, B, N, F, T)
    Y, status = plan.auxiva_from_stft(torch.from_numpy(X).to(device), num_epochs=epochs)
    assert not status.cpu().numpy().any()
    Y = Y.cpu().numpy()
    assert Y.dtype == np.complex128 and Y.shape == X.shape
    worst = 0.0
    for b in (range(B) if check is None else check):
        want = ao.auxiva(X[b].transpose(0, 2, 1), epochs).transpose(0, 2, 1)
        err = rel_err(Y[b], want)
        assert err <= TOL, f"N={N} epochs={epochs} b={b}: {err:.3e} of max|Y|"
        worst = max(worst, err)
    return worst


def run_fixtures(device):
    """The kernels on the reference's inputs against the reference's own Y (every 32nd bin)."""
    from setk_b200 import plan
    g = load_fixture()
    worst = {}
    for name in NAMES:
        X = fixture_stft(g[name + "/pcm16"])                                    # N x T x F
        x = torch.from_numpy(np.ascontiguousarray(X.transpose(0, 2, 1))[None]).to(device)
        Y, status = plan.auxiva_from_stft(x, num_epochs=EPOCHS)
        assert int(status[0]) == 0
        got = Y[0].cpu().numpy().transpose(0, 2, 1)[:, :, ::BIN_STEP]
        want = g[name + "/Y_bins"]
        worst[name] = rel_err(got, want)
        assert worst[name] <= TOL, f"{name}: {worst[name]:.3e} of max|Y|"
    return worst


def write_cli_inputs(tmp_path, with_silent=True):
    """wav.scp of the fixtures, plus (with_silent) a key whose second channel is silent: W^H V is
    exactly singular there and the reference would die with LinAlgError."""
    import scipy.io.wavfile as wavfile
    g = load_fixture()
    lines = []
    for name in NAMES:
        wavfile.write(str(tmp_path / f"{name}.wav"), 16000, g[name + "/pcm16"].T)
        lines.append(f"{name} {tmp_path / (name + '.wav')}")
    if with_silent:
        pcm = g["mix2/pcm16"].copy()
        pcm[1] = 0
        wavfile.write(str(tmp_path / "silent.wav"), 16000, pcm.T)
        lines.insert(1, f"silent {tmp_path / 'silent.wav'}")
    (tmp_path / "wav.scp").write_text("\n".join(lines) + "\n")
    return g


def check_cli(tmp_path, library=None):
    """Every source file within 1 LSB of the reference's; the silent-channel key skipped, the run goes on."""
    import scipy.io.wavfile as wavfile
    g = write_cli_inputs(tmp_path)
    out = tmp_path / "out"
    run_script("apply_auxiva.py", [str(tmp_path / "wav.scp"), str(out)], library)
    assert not list(out.glob("silent.*")), "the singular utterance was written"
    stats = {}
    for name in NAMES:
        want = g[name + "/cli_pcm16"]
        for idx in range(want.shape[0]):
            sr, got = wavfile.read(str(out / f"{name}.src{idx + 1}.wav"))
            assert sr == 16000 and got.dtype == np.int16 and got.shape == want[idx].shape
            d = np.abs(got.astype(np.int32) - want[idx].astype(np.int32))
            assert d.max() <= 1, f"{name}.src{idx + 1}: {d.max()} LSB"
            stats[f"{name}.src{idx + 1}"] = float(np.mean(d == 0))
    assert not (out / f"{name}.src{want.shape[0] + 1}.wav").exists()
    return stats
