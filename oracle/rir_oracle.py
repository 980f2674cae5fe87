"""
Float64 restatement of the reference's image-method RIR generator (include/rir-generator.cc:25-223,
rir-generator.h:156-169: Habets' RIR-Generator as rir-simulate runs it), vectorised over the image
lattice.  Test infrastructure: the kernel (csrc/rir.cu) is checked against this, and this against
the reference's own generator compiled by oracle/rir_ref/build.sh.

Every step is the reference's, in float64 where the reference uses float32:
  * positions scaled to samples by cts = c / fs; Tw = 2 int(0.004 fs + 0.5);
  * lattice x in [-nx, nx], nx = ceil(L / (2 Tx)), and so on, times mirror bits q, j, k;
  * reflection factor b0^|x-q| b1^|x| b2^|y-j| b3^|y| b4^|z-k| b5^|z| (0^0 = 1);
  * kept when |2x-q| + |2y-j| + |2z-k| <= order (or order == -1) and floor(dist) < L;
  * Tw taps from floor(dist) - Tw/2 + 1: gain 0.5 (1 - cos(2 pi (n+1-frac)/Tw)) sinc(pi (n+1-frac-Tw/2)),
    gain = mic * refl / (4 pi dist cts); taps outside [0, L) dropped;
  * MicrophoneSim with acos / atan2 as written (rir-generator.cc:194-223);
  * the optional 2-pole 100 Hz high-pass over the channel (rir-generator.cc:180-190).
"""
import math

import numpy as np

MIC_RHO = {"omnidirectional": 1.0, "subcardioid": 0.75, "cardioid": 0.5, "hypercardioid": 0.25,
           "bidirectional": 0.0}
MIC_TYPES = tuple(MIC_RHO)


def window_taps(fs):
    """Tw of rir-generator.cc:119"""
    return 2 * int(0.004 * fs + 0.5)


def t60_to_beta(room, t60, c):
    """rir-generator.cc:78-92: six equal coefficients from one T60; T60 = 0 gives beta = 0"""
    lx, ly, lz = (float(v) for v in room)
    if t60 == 0:
        return np.zeros(6)
    V, S = lx * ly * lz, 2 * (lx * ly + lx * lz + ly * lz)
    alpha = 24 * V * math.log(10.0) / (c * S * t60)
    if alpha > 1:
        raise ValueError(f"{alpha} > 1: The reflection coefficients cannot be calculated using the current "
                         "room parameters, i.e. room size and reverberation time.")
    return np.full(6, math.sqrt(1 - alpha))


def _lattice(L, T):
    n = [int(math.ceil(L / (2 * t))) for t in T]
    x, y, z, q, j, k = np.meshgrid(np.arange(-n[0], n[0] + 1), np.arange(-n[1], n[1] + 1),
                                   np.arange(-n[2], n[2] + 1), [0, 1], [0, 1], [0, 1], indexing="ij")
    return [v.ravel() for v in (x, y, z, q, j, k)]


def mic_gain(p, dist, rho, azimuth, elevation):
    """MicrophoneSim (rir-generator.cc:194-223), p = the image's offset in samples"""
    if rho == 1:
        return np.ones_like(dist)
    theta = np.arccos(p[2] / dist)
    phi = np.arctan2(p[1], p[0])
    g = (np.sin(np.pi / 2 - elevation) * np.sin(theta) * np.cos(azimuth - phi) +
         np.cos(np.pi / 2 - elevation) * np.cos(theta))
    return rho + (1 - rho) * g


def high_pass(h, fs):
    """rir-generator.cc:180-190 in float64"""
    W = 2 * math.pi * 100 / fs
    R1 = math.exp(-W)
    B1, B2, A1 = 2 * R1 * math.cos(W), -R1 * R1, -1 - R1
    out = np.empty_like(h)
    y1 = y2 = 0.0
    for i, x0 in enumerate(h.tolist()):
        y0 = B1 * y1 + B2 * y2 + x0
        out[i] = y0 + A1 * y1 + R1 * y2
        y2, y1 = y1, y0
    return out


def rir(room, beta, source, receivers, n_samples, fs=16000, c=340, order=-1, mic_type="omnidirectional",
        orientation=(0, 0), hp_filter=True):
    """
    One problem: room (3,), beta (6,) reflection coefficients, source (3,), receivers (M, 3), metres.
    Returns (M, L) float64.
    """
    L = int(n_samples)
    cts = c / fs
    Tw = window_taps(fs)
    T = np.asarray(room, np.float64) / cts
    S = np.asarray(source, np.float64) / cts
    beta = np.asarray(beta, np.float64)
    rho = MIC_RHO[mic_type]
    az, el = (float(v) for v in orientation)
    x, y, z, q, j, k = _lattice(L, T)
    keep = np.ones(x.shape, bool) if order == -1 else (
        np.abs(2 * x - q) + np.abs(2 * y - j) + np.abs(2 * z - k) <= order)
    x, y, z, q, j, k = (v[keep] for v in (x, y, z, q, j, k))
    with np.errstate(divide="ignore", invalid="ignore"):
        refl = (beta[0]**np.abs(x - q) * beta[1]**np.abs(x) * beta[2]**np.abs(y - j) * beta[3]**np.abs(y) *
                beta[4]**np.abs(z - k) * beta[5]**np.abs(z))
    n = np.arange(Tw)
    out = np.zeros((len(receivers), L))
    for m, rcv in enumerate(np.asarray(receivers, np.float64)):
        R = rcv / cts
        p = np.stack([(1 - 2 * q) * S[0] - R[0] + 2 * x * T[0], (1 - 2 * j) * S[1] - R[1] + 2 * y * T[1],
                      (1 - 2 * k) * S[2] - R[2] + 2 * z * T[2]])
        dist = np.sqrt(np.sum(p * p, axis=0))
        fdist = np.floor(dist)
        sel = fdist < L
        d, fd, pr, rf = dist[sel], fdist[sel], p[:, sel], refl[sel]
        gain = mic_gain(pr, d, rho, az, el) * rf / (4 * np.pi * d * cts)
        for i in range(0, len(d), 8192):
            frac = (d[i:i + 8192] - fd[i:i + 8192])[:, None]
            u = n[None, :] + 1 - frac - Tw // 2
            with np.errstate(divide="ignore", invalid="ignore"):
                sinc = np.where(u == 0, 1.0, np.sin(np.pi * u) / (np.pi * u))
            taps = gain[i:i + 8192, None] * 0.5 * (1 - np.cos(2 * np.pi * (n[None, :] + 1 - frac) / Tw)) * sinc
            idx = fd[i:i + 8192].astype(np.int64)[:, None] - Tw // 2 + 1 + n[None, :]
            ok = (idx >= 0) & (idx < L)
            out[m] += np.bincount(idx[ok], weights=taps[ok], minlength=L)
        if hp_filter:
            out[m] = high_pass(out[m], fs)
    return out


def peak_err(got, want):
    """max |got - want| over each channel's peak |want|, the worst channel (..., L)"""
    got = np.asarray(got, np.float64).reshape(-1, np.shape(want)[-1])
    want = np.asarray(want, np.float64).reshape(got.shape)
    return float(np.max(np.max(np.abs(got - want), axis=1) / np.max(np.abs(want), axis=1)))
