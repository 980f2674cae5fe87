"""
oracle/feats_oracle.py -- CPU restatement of the reference's spectral feature command lines.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Not imported by the product.

What it restates
  * scripts/sptk/compute_spectrogram.py:19-40  SpectrogramReader(apply_abs=True, ...) -> channel 0,
    T x F float32; samples always int16 / 32768 (--normalize-samples is parsed and never passed on)
  * scripts/sptk/compute_fbank.py:22-61        np.dot(mel, |X|) of channel 0 -> T x N, optional
    log(max(., EPSILON)); samples int16 values unless --normalize-samples true
and librosa 0.8.1 `filters.mel` (htk=True, norm="slaney", float32), which is not in the reference
tree, in its own copy (mel() below), so that the product's setk_b200.libs.filters is checked
against an independent statement.  The STFT is oracle/stft_oracle.py's forward_stft in complex64.

Pinned by: oracle/make_golden_feats.py runs the reference's own scripts on the doc assets under
oracle/ref_shim.py with mel() standing in for librosa.filters.mel (tests/golden/ref_feats.npz).
"""
import warnings

import numpy as np

from . import stft_oracle as so

EPSILON = so.EPSILON


def mel(sr, n_fft, n_mels=128, fmin=0.0, fmax=None, htk=False, norm="slaney", dtype=np.float32):
    """librosa 0.8.1 filters.mel, the htk=True / norm="slaney" branch the reference reaches."""
    assert htk and norm == "slaney", "only htk=True, norm='slaney' is restated"
    if fmax is None:
        fmax = float(sr) / 2
    n_mels = int(n_mels)
    weights = np.zeros((n_mels, int(1 + n_fft // 2)), dtype=dtype)
    fftfreqs = np.linspace(0, float(sr) / 2, int(1 + n_fft // 2), endpoint=True)   # fft_frequencies
    lo, hi = (2595.0 * np.log10(1.0 + np.asanyarray(f) / 700.0) for f in (fmin, fmax))   # hz_to_mel
    mel_f = 700.0 * (10.0**(np.linspace(lo, hi, n_mels + 2) / 2595.0) - 1.0)              # mel_frequencies
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
    weights *= enorm[:, np.newaxis]
    if not np.all((mel_f[:-2] == 0) | (weights.max(axis=1) > 0)):
        warnings.warn("Empty filters detected in mel frequency basis. "
                      "Some channels will produce empty responses. "
                      "Try increasing your sampling rate (and fmax) or "
                      "reducing n_mels.")
    return weights


def _stft_kwargs(o):
    return dict(frame_len=o["frame_len"], frame_hop=o["frame_hop"], round_power_of_two=o["round_power_of_two"],
                window=o["window"], center=o["center"], out_dtype=np.complex64)


def spectrogram(pcm, o):
    """compute_spectrogram.py of channel 0 of int16 samples pcm (C x N or N): T x F float32."""
    x = so.float_from_pcm16(np.atleast_2d(pcm)[0])
    return so.forward_stft(x, apply_abs=True, apply_log=o["apply_log"], apply_pow=o["apply_pow"],
                           transpose=True, **_stft_kwargs(o))


def fbank(pcm, o, linear=False):
    """
    compute_fbank.py of channel 0 of int16 samples pcm: T x N float32.  linear=True returns the mel
    projection before the log (the value the log tolerance is stated on).
    """
    x = np.atleast_2d(pcm)[0]
    x = so.float_from_pcm16(x) if o["normalize"] else x.astype(np.float32)
    spec = so.forward_stft(x, apply_abs=True, transpose=False, **_stft_kwargs(o))    # F x T
    n_fft = so.nextpow2(o["frame_len"]) if o["round_power_of_two"] else o["frame_len"]
    weights = mel(o["sr"], n_fft, n_mels=o["num_bins"], fmin=o["min_freq"], fmax=o["max_freq"], htk=True)
    fb = np.transpose(np.dot(weights, spec))
    if o["apply_log"] and not linear:
        fb = np.log(np.maximum(fb, EPSILON))
    return fb


SPECTROGRAM_DEFAULTS = dict(frame_len=512, frame_hop=256, round_power_of_two=True, window="hann", center=True,
                            apply_log=False, apply_pow=False)
FBANK_DEFAULTS = dict(frame_len=512, frame_hop=256, round_power_of_two=True, window="hann", center=True,
                      apply_log=False, normalize=False, sr=16000, num_bins=40, min_freq=0, max_freq=8000)


def parse_flags(script, flags):
    """The options of a fixture run's flag list, with the script's defaults (StftParser's included)."""
    o = dict(SPECTROGRAM_DEFAULTS if script == "compute_spectrogram.py" else FBANK_DEFAULTS)
    i = 0
    while i < len(flags):
        k, v = flags[i][2:].replace("-", "_"), flags[i + 1]
        k = {"normalize_samples": "normalize"}.get(k, k)
        if k in ("frame_len", "frame_hop", "sr", "num_bins", "min_freq", "max_freq"):
            o[k] = int(v)
        elif k in ("round_power_of_two", "center", "apply_log", "apply_pow", "normalize"):
            o[k] = v.lower() in ("true", "1", "yes", "y", "t", "on")
        elif k == "window":
            o[k] = v
        i += 2
    if script == "compute_spectrogram.py":
        o.pop("normalize", None)      # parsed and never passed on: samples are always int16 / 32768
    return o


def run(script, pcm, flags):
    """The oracle's features of one utterance for a fixture run."""
    o = parse_flags(script, flags)
    return spectrogram(pcm, o) if script == "compute_spectrogram.py" else fbank(pcm, o)
