"""
oracle/simu_oracle.py -- a float64 numpy restatement of the reference's wav_simulate.py run_simu
(scripts/sptk/wav_simulate.py:17-312), written for the tests of csrc/simu.cu and setk_b200/simu.py.

simulate(args, read) returns (mix, [speaker references], noise reference or None) in float64, for an
argparse namespace with wav_simulate.py's flags; `read(path, beg, end, sr)` returns what read_wav
returns (C x N or N float32).  dtype=np.float32 runs the convolutions in float32 as the reference's
scipy does (the CPU line of tools/bench_simu.py).  The reference's errors are raised as it raises
them; where its point-noise mixing loop's numpy broadcast fails, ValueError.
"""
import numpy as np
import scipy.signal as ss

EPS32 = float(np.finfo(np.float32).eps)


def coeff_snr(sig_pow, ref_pow, snr):
    return (ref_pow / (sig_pow * 10**(snr / 10) + EPS32))**0.5


def room_image(src, rir, channel, dtype=np.float64):
    """each selected RIR channel convolved with the mono source, truncated to the source's length"""
    if src.ndim != 1:
        raise RuntimeError(f"Can not convolve rir with {src.ndim}D signals")
    rir = rir[None] if rir.ndim == 1 else rir
    if channel >= 0:
        rir = rir[channel:channel + 1]
    if rir.shape[0] == 0:
        raise ValueError("no RIR channel selected")
    out = ss.fftconvolve(src[None].astype(dtype), rir.astype(dtype), axes=-1)[:, :src.size]
    return out.astype(np.float64)


def _floats(s):
    return [float(v) for v in s.split(",")] if s else None


def _load(paths, read, sr, beg=None, end=None):
    if not paths:
        return None
    p = paths.split(",")
    b = [int(v) for v in beg.split(",")] if beg else [None] * len(p)
    e = [int(v) for v in end.split(",")] if end else [None] * len(p)
    return [read(f, b_, e_, sr) for f, b_, e_ in zip(p, b, e)]


def simulate(a, read, dtype=np.float64):
    spks = _load(a.src_spk, read, a.sr)
    rirs = _load(a.src_rir, read, a.sr)
    if rirs and len(rirs) != len(spks):
        raise RuntimeError("Number of --src-rir do not match with --src-spk option")
    sdr = _floats(a.src_sdr)
    if len(spks) > 1 and not sdr:
        raise RuntimeError("--src-sdr need to be assigned")
    if sdr:
        if len(sdr) != len(spks) - 1:
            raise RuntimeError("Number of --src-snr - 1 do not match with --src-snr option")
        sdr = [0.0] + sdr
    begin = [int(v) for v in _floats(a.src_begin)] if a.src_begin else [0] * len(spks)
    T = max(b + s.size for b, s in zip(begin, spks))

    noise_rirs = _load(a.point_noise_rir, read, a.sr)
    offs = a.point_noise_offset.split()
    noises = _load(a.point_noise, read, a.sr, beg=a.point_noise_offset, end=",".join(str(int(v) + T) for v in offs))
    if a.point_noise:
        if noise_rirs and len(noises) != len(noise_rirs):
            raise RuntimeError("Number of --point-noise-rir do not match with --point-noise option")
        snr = _floats(a.point_noise_snr)
        if not snr:
            raise RuntimeError("--point-noise-snr need to be assigned")
        if len(snr) != len(noises):
            raise RuntimeError("Number of --point-noise-snr do not match with --point-noise option")
        nbeg = [int(v) for v in _floats(a.point_noise_begin)] if a.point_noise_begin else [0] * len(noises)
    iso = _load(a.isotropic_noise, read, a.sr, beg=str(a.isotropic_noise_offset),
                end=str(a.isotropic_noise_offset + T))
    if iso:
        iso = iso[0]
        iso_snr = _floats(a.isotropic_noise_snr)
        if not iso_snr:
            raise RuntimeError("--isotropic-snr need to be assigned")
        iso_snr = iso_snr[0]

    ch = a.dump_channel
    images = []
    for i, s in enumerate(spks):
        img = (s[None] if s.ndim == 1 else s).astype(np.float64) if rirs is None else room_image(s, rirs[i], ch, dtype)
        images.append(img)
    N = images[0].shape[0]
    p0 = np.mean(images[0][0]**2)
    spk = []
    for i, img in enumerate(images):
        c = 1.0 if i == 0 else coeff_snr(np.mean(img[0]**2), p0, sdr[i])
        buf = np.zeros((N, T))
        buf[:, begin[i]:begin[i] + img.shape[-1]] += c * img
        spk.append(buf)
    spk_sum = sum(spk)
    p_spk = np.mean(spk_sum[0]**2)
    mix, noise = spk_sum.copy(), None
    if noises:
        imgs, pows, durs = [], [], []
        for i, n in enumerate(noises):
            b = nbeg[i]
            if not a.point_noise_repeat:
                dur = min(n.shape[-1], T - b)
            else:
                dur = T - b
                if n.shape[-1] < dur:
                    n = np.pad(n, (0, dur - n.shape[-1]), mode="wrap")
            if noise_rirs is None:
                img = (n[None] if n.ndim == 1 else n).astype(np.float64)
                pows.append(np.mean(img[0, :dur]**2))
            else:
                img = room_image(n[:dur], noise_rirs[i], ch, dtype)
                pows.append(np.mean(img[0]**2))
            imgs.append(img)
            durs.append(dur)
        dur = durs[-1]
        noise = np.zeros((imgs[0].shape[0], T))
        for i, img in enumerate(imgs):
            b = nbeg[i]
            noise[..., b:b + dur] += coeff_snr(pows[i], p_spk, snr[i]) * img[..., :dur]   # numpy may raise
        if noise.shape[0] != N:
            raise RuntimeError(f"Channel mismatch between source speaker configuration and pointsource noise's, "
                               f"{N} vs {noise.shape[0]}")
        mix = spk_sum + noise
    if iso is not None:
        if N == 1:
            if iso.ndim == 1:
                iso = iso[None]
            elif ch >= 0:
                iso = iso[ch:ch + 1]
            else:
                raise RuntimeError("Single channel mixture vs multi-channel isotropic noise")
        elif iso.shape[0] != N:
            raise RuntimeError(f"Channel number mismatch between mixture and isotropic noise, {N} vs {iso.shape[0]}")
        dur = min(T, iso.shape[-1])
        chunk = iso[0, :dur].astype(np.float64)
        c = coeff_snr(np.mean(chunk**2), p_spk, iso_snr)
        mix[..., :dur] += c * chunk
        if noise is None:
            noise = np.zeros((N, T))   # the reference keeps coeff * chunk alone (see setk_b200/simu.py)
        noise[..., :dur] += c * chunk
    factor = a.norm_factor / (np.max(np.abs(mix)) + EPS32)
    return mix.squeeze() * factor, [s[0] * factor for s in spk], None if noise is None else noise[0] * factor
