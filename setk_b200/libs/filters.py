"""
setk_b200.libs.filters -- the mel filterbank compute_fbank.py builds (compute_fbank.py:45-48:
librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax, htk=True)), on the host in numpy, so that the
package needs no librosa.  setk_plan_set_mel (StftPlan.set_mel) takes the result.
"""
import warnings

import numpy as np


def hz_to_mel(frequencies, htk=False):
    """librosa 0.8.1 core.convert.hz_to_mel, HTK scale only."""
    if not htk:
        raise ValueError("only the HTK mel scale (htk=True) is implemented")
    return 2595.0 * np.log10(1.0 + np.asanyarray(frequencies) / 700.0)


def mel_to_hz(mels, htk=False):
    """librosa 0.8.1 core.convert.mel_to_hz, HTK scale only."""
    if not htk:
        raise ValueError("only the HTK mel scale (htk=True) is implemented")
    return 700.0 * (10.0**(np.asanyarray(mels) / 2595.0) - 1.0)


def mel(sr, n_fft, n_mels=128, fmin=0.0, fmax=None, htk=False, norm="slaney", dtype=np.float32):
    """
    librosa 0.8.1 filters.mel: n_mels x (1 + n_fft // 2) triangular filters on the mel scale, each
    scaled to unit area (norm="slaney").  The ramps are float64 and stored into `dtype`, then scaled
    in place, as librosa does.  Only what the reference reaches is implemented, htk=True with
    norm="slaney"; anything else raises ValueError.  Filters that no FFT bin reaches come out as zero
    rows, with librosa's "Empty filters detected" UserWarning.
    """
    if not htk:
        raise ValueError("only the HTK mel scale (htk=True) is implemented")
    if norm != "slaney":
        raise ValueError(f"only norm='slaney' is implemented, got {norm!r}")
    if fmax is None:
        fmax = float(sr) / 2
    n_mels = int(n_mels)
    weights = np.zeros((n_mels, int(1 + n_fft // 2)), dtype=dtype)
    fftfreqs = np.linspace(0, float(sr) / 2, int(1 + n_fft // 2), endpoint=True)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(fmin, htk=True), hz_to_mel(fmax, htk=True), n_mels + 2), htk=True)
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
