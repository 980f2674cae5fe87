"""
Spectral features: the cases and checks shared by the CPU tier (tests/test_feats.py, kernels on the CPU
execution model) and the GPU tier (tests/test_gpu_feats.py).
"""
import json
import os

import numpy as np
import torch

from oracle import feats_oracle as fo
from oracle import stft_oracle as so

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL_LIN = 2e-5      # per-utterance rel-inf of linear outputs (magnitude, fbank): the STFT's TOL_F32
TOL_POW = 4e-5      # power
TOL_LOG = 2e-3      # |delta| of log outputs where the oracle's linear value is >= 1e-2 of its maximum


def fixture():
    return np.load(os.path.join(GOLD, "ref_feats.npz"))


def fixture_runs(g):
    return sorted({k.split("/")[0] for k in g.files if not k.startswith("in/")})


def run_info(g, name):
    return str(g[f"{name}/script"]), json.loads(str(g[f"{name}/keys"])), json.loads(str(g[f"{name}/flags"]))


def compare(got, lin_ref, log, pw=False):
    """
    Worst errors of features `got` against the oracle's linear values lin_ref (same shape): the linear
    rel-inf (of max(v, EPSILON) for log outputs) and, for log outputs, the largest |delta| on entries
    >= 1e-2 of the maximum.  Asserts the tolerances; returns (rel, dlog).
    """
    got = np.asarray(got, dtype=np.float64)
    lin_ref = np.asarray(lin_ref, dtype=np.float64)
    assert got.shape == lin_ref.shape, (got.shape, lin_ref.shape)
    peak = max(np.max(np.abs(lin_ref)), 1e-30)
    if log:
        lin_got = np.exp(got)
        lin_ref_c = np.maximum(lin_ref, fo.EPSILON)
        rel = np.max(np.abs(lin_got - lin_ref_c)) / max(np.max(lin_ref_c), 1e-30)
        big = lin_ref >= 1e-2 * peak
        dlog = float(np.max(np.abs(got - np.log(lin_ref_c))[big])) if big.any() else 0.0
        assert dlog <= TOL_LOG, dlog
    else:
        rel = np.max(np.abs(got - lin_ref)) / peak
        dlog = 0.0
    assert rel <= (TOL_POW if pw else TOL_LIN), rel
    return float(rel), dlog


def oracle_linear(x, fl, hop, center, rp2, window, pw=False, weights=None, scale=1.0):
    """Oracle features of every channel of x (C x N float32) before any log: C x T x D float64."""
    out = []
    for c in range(x.shape[0]):
        S = so.forward_stft(x[c], frame_len=fl, frame_hop=hop, round_power_of_two=rp2, center=center,
                            window=window, transpose=False, out_dtype=np.complex64)
        m = so.cmat_abs(S).astype(np.float64) * scale
        if pw:
            m = m * m
        if weights is not None:
            m = weights.astype(np.float64) @ m
        out.append(m.T)
    return np.stack(out)


def check_plan(device, rng, C, fl, hop, center, window="hann", rp2=True, lens=(3000,), n_mels=None, pw=False,
               log=False):
    """StftPlan.spectral_feats on a ragged batch against the oracle; frames past a length are zero rows."""
    from setk_b200 import plan as P
    from setk_b200.libs.filters import mel
    N = max(lens)
    B = len(lens)
    x = np.zeros((B, C, N), np.float32)
    for b, n in enumerate(lens):
        x[b, :, :n] = rng.standard_normal((C, n)).astype(np.float32) * 0.3
    pl = P.StftPlan(C, fl, hop, center, rp2, window, B, N, device)
    weights = None
    if n_mels:
        weights = mel(16000, pl.n_fft, n_mels=n_mels, htk=True)
        pl.set_mel(weights)
    ns = torch.tensor(lens, dtype=torch.int32) if B > 1 else None
    out = pl.spectral_feats(torch.from_numpy(x).to(device), n_samples=ns, apply_pow=pw, mel=bool(n_mels),
                            apply_log=log).cpu().numpy()
    worst = (0.0, 0.0)
    for b, n in enumerate(lens):
        ref = oracle_linear(x[b, :, :n], fl, hop, center, rp2, window, pw, weights)
        Tb = ref.shape[1]
        r = compare(out[b, :, :Tb], ref, log, pw)
        worst = tuple(max(u, v) for u, v in zip(worst, r))
        assert not out[b, :, Tb:].any()
    pl.close()
    return worst


def fixture_features(device, g, name, key):
    """The product's features of one fixture utterance through StftPlan, as the script computes them."""
    from setk_b200 import plan as P
    from setk_b200.libs.filters import mel
    script, _, flags = run_info(g, name)
    o = fo.parse_flags(script, flags)
    pcm = np.atleast_2d(g[f"in/{key}"])[0]
    N = pcm.shape[-1]
    pl = P.StftPlan(1, o["frame_len"], o["frame_hop"], o["center"], o["round_power_of_two"], o["window"], 1, N,
                    device)
    x = torch.from_numpy(pcm.astype(np.float32) / np.float32(32768.0)).view(1, 1, N).to(device)
    if script == "compute_spectrogram.py":
        out = pl.spectral_feats(x, apply_pow=o["apply_pow"], apply_log=o["apply_log"])
        lin = fo.spectrogram(pcm, dict(o, apply_log=False))
        pw = o["apply_pow"]
    else:
        pl.set_mel(mel(o["sr"], pl.n_fft, n_mels=o["num_bins"], fmin=o["min_freq"], fmax=o["max_freq"], htk=True))
        out = pl.spectral_feats(x, mel=True, apply_log=o["apply_log"], sample_scale=1.0 if o["normalize"] else 32768.0)
        lin = fo.fbank(pcm, o, linear=True)
        pw = False
    pl.close()
    return out[0, 0].cpu().numpy(), lin, o["apply_log"], pw
