"""
Shared cases of the noise-suppression tests (tests/test_ns.py on the CPU execution model,
tests/test_gpu_ns.py on the device): setk_ns_imcra through setk_b200.plan.ns_from_stft against the
float64 oracle (oracle/ns_oracle.py) and the reference fixtures (tests/golden/ref_ns.npz), and
scripts/sptk/apply_ns.py against the reference's shipped output.
"""
import os

import numpy as np
import torch

from script_runner import run_script

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_ns.npz")

from oracle import ns_oracle as no  # noqa: E402
from oracle import stft_oracle  # noqa: E402

FRAME_STEP = 8
STFT_KW = dict(frame_len=512, frame_hop=256, window="hann", center=True, round_power_of_two=True)
CASE_B_CONF = dict(U=20, V=7, w_mcra=2, h_mcra="hamming", alpha=0.9, beta=1.2, gamma0=5.0, gmin_db=-15)
# gain against the float64 oracle: |dG| <= TOL_GAIN max(1, |G|); enh relative to max |enh|
TOL_GAIN = 1e-9
TOL_ENH = 1e-6
# the oracle and the kernels against the reference's stored gains (quad's own tolerance is 1.49e-8,
# and the reference squares |x| in float32): observed 3.9e-7 on the clip, 2.4e-7 on case b
TOL_REF = 1e-6


def load_fixture():
    return dict(np.load(GOLD))


def fixture_stft(pcm):
    """T x F complex64 STFT of PCM-16 audio, as the reference's SpectrogramReader computes it."""
    return stft_oracle.forward_stft(stft_oracle.float_from_pcm16(pcm), transpose=True, out_dtype=np.complex64,
                                    **STFT_KW)


def noisy_stft(rng, B, F, T, silence=True):
    """B x F x T complex64: noise under a bursty envelope; with `silence` utterance 0 starts with an
    all-zero frame, has an all-zero bin and a zero run in the middle."""
    env = 0.05 + rng.gamma(0.6, 1.0, (B, 1, T)) * (rng.random((B, 1, T)) < 0.5)
    X = ((rng.standard_normal((B, F, T)) + 1j * rng.standard_normal((B, F, T))) * (0.02 + env)).astype(np.complex64)
    if silence:
        X[0, :, 0] = 0
        X[0, F // 3, :] = 0
        X[0, :, T // 2:T // 2 + 5] = 0
    return X


def gain_err(got, want):
    return float(np.max(np.abs(got - want) / np.maximum(1.0, np.abs(want))))


def enh_err(got, want):
    return float(np.max(np.abs(got - want)) / max(np.max(np.abs(want)), 1e-30))


def run_parity(device, B, F, T, conf, rng, check=None, n_frames=None):
    """plan.ns_from_stft against the float64 oracle on utterances `check` (default: all)."""
    from setk_b200 import plan
    X = noisy_stft(rng, B, F, T)
    g, e = plan.ns_from_stft(torch.from_numpy(X).to(device), n_frames=n_frames, config=conf)
    g, e = g.cpu().numpy(), e.cpu().numpy()
    assert g.dtype == np.float64 and g.shape == (B, T, F) and e.shape == (B, F, T)
    worst = (0.0, 0.0)
    for b in (range(B) if check is None else check):
        nf = None if n_frames is None else [n_frames[b]]
        go, eo = no.ns_bft(X[b:b + 1], nf, **conf)
        eg, ee = gain_err(g[b], go[0]), enh_err(e[b], eo[0])
        assert eg <= TOL_GAIN, f"F={F} T={T} {conf} b={b}: gain {eg:.3e}"
        assert ee <= TOL_ENH, f"F={F} T={T} {conf} b={b}: enh {ee:.3e} of max|enh|"
        worst = (max(worst[0], eg), max(worst[1], ee))
    return worst


def run_cases(device):
    """The kernels on the reference's stored cases (a) silence and (b) a non-default configuration."""
    from setk_b200 import plan
    gold = load_fixture()
    worst = {}
    for name, conf in (("a", {}), ("b", CASE_B_CONF)):
        S = gold[name + "/stft"]                                                     # T x F
        g, _ = plan.ns_from_stft(torch.from_numpy(np.ascontiguousarray(S.T))[None].to(device), config=conf,
                                 enh=False)
        g = g[0].cpu().numpy()
        go = no.iMCRA(**conf).run(S)
        assert gain_err(g, go) <= TOL_GAIN, name
        worst[name] = gain_err(g, gold[name + "/gain"])
        assert worst[name] <= TOL_REF, f"{name}: {worst[name]:.3e} against the reference"
        assert np.all(np.isfinite(g))
    return worst


def run_clip(device):
    """The kernels on the doc clip against the reference's gains (every 8th frame)."""
    from setk_b200 import plan
    gold = load_fixture()
    X = fixture_stft(gold["egs/pcm16"])                                             # T x F
    g, _ = plan.ns_from_stft(torch.from_numpy(np.ascontiguousarray(X.T))[None].to(device), enh=False)
    err = float(np.max(np.abs(g[0].cpu().numpy()[::FRAME_STEP] - gold["egs/gain_frames"])))
    assert err <= TOL_REF, f"clip: {err:.3e}"
    return err


def write_cli_inputs(tmp_path, with_multichannel=True):
    """wav.scp of the doc clip, plus (with_multichannel) a 2-channel key the port skips."""
    import scipy.io.wavfile as wavfile
    gold = load_fixture()
    pcm = gold["egs/pcm16"]
    wavfile.write(str(tmp_path / "egs.wav"), 16000, pcm)
    lines = [f"egs {tmp_path / 'egs.wav'}"]
    if with_multichannel:
        wavfile.write(str(tmp_path / "stereo.wav"), 16000, np.stack([pcm, pcm[::-1]], 1))
        lines.insert(0, f"stereo {tmp_path / 'stereo.wav'}")
    (tmp_path / "wav.scp").write_text("\n".join(lines) + "\n")
    return gold


def check_cli(tmp_path, library=None):
    """--output wave: every sample within 1 LSB of the shipped egs_ns.wav, >= 99 % exact; the
    multichannel key skipped.  Returns the exact fraction."""
    import scipy.io.wavfile as wavfile
    gold = write_cli_inputs(tmp_path)
    out = tmp_path / "out"
    run_script("apply_ns.py", [str(tmp_path / "wav.scp"), str(out)], library)
    assert not list(out.glob("stereo.*")), "the multichannel key was written"
    sr, got = wavfile.read(str(out / "egs.wav"))
    want = gold["egs/ns_pcm16"]
    assert sr == 16000 and got.dtype == np.int16 and got.shape == want.shape
    d = np.abs(got.astype(np.int32) - want.astype(np.int32))
    assert d.max() <= 1, f"{d.max()} LSB"
    exact = float(np.mean(d == 0))
    assert exact >= 0.99, exact
    return exact
