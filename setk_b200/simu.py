"""
setk_b200.simu -- speech + RIR + noise mixtures in device batches (the reference's
scripts/sptk/wav_simulate.py, run_simu at wav_simulate.py:166-312).

plan_mixture(args) restates run_simu's host bookkeeping for one invocation: audio loading, begins,
durations, repeat padding, channel selection and the reference's errors.  It returns a Mixture: the
convolutions to run and the terms to mix.  simulate(mixtures, device) groups mixtures into device
batches under a memory budget, runs every convolution of a batch through setk_convolve (one call per
channel count) and the mixing through setk_simulate_mix, and returns each mixture's outputs.

Kept quirks of the reference (each one changes results or errors, so it is reproduced):
  * mix_nsamps = max(begin + source.size): the size of a multichannel source counts all its channels.
  * The point-noise mixing loop uses the last noise's duration for every noise (:141-142).  Where that
    still gives a result (the same length, or a one-sample image broadcast) it is reproduced; where
    numpy's broadcast fails, ValueError names the mixture.
  * The isotropic noise's channel 0 alone is added to every channel, at the power of that channel;
    the file must still have the mixture's channel count (or one channel for a one-channel mixture).
  * --point-noise-offset is split on whitespace, so it holds one offset, and zip() then reads only as
    many noise files as offsets.
  * --point-noise-repeat pads with numpy's wrap mode on every axis of the noise.
  * Powers are taken on channel 0 only.
Deviation: with an isotropic noise and no point noise the reference's noise reference is a scalar and
writing it fails; here it is the isotropic noise's channel-0 track.
"""
import os
from dataclasses import dataclass, field

import numpy as np
import torch

from . import _lib, plan
from .libs.utils import read_wav

# device memory for one batch: pool of images, spectra of the convolutions and outputs
BATCH_BYTES = 1 << 30


@dataclass
class Conv:
    x: object            # (S,) source, numpy float32 or a tensor
    h: object            # (M, L) filter
    n_out: int


@dataclass
class Term:
    kind: int            # _lib.SIMU_*
    image: object        # (C, T) array / tensor, or a Conv whose output is the image
    begin: int
    length: int
    repeat: int
    power: tuple         # (begin, end) on channel 0
    level: float

    def channels(self):
        return self.image.h.shape[0] if isinstance(self.image, Conv) else self.image.shape[0]

    def samples(self):
        return self.image.n_out if isinstance(self.image, Conv) else self.image.shape[-1]


@dataclass
class Mixture:
    name: str
    n_samples: int
    n_channels: int
    norm_factor: float
    terms: list = field(default_factory=list)

    def n_speakers(self):
        return sum(t.kind == _lib.SIMU_SPEAKER for t in self.terms)


def _load_audio(src_args, beg=None, end=None, sr=16000, read=read_wav):
    """load_audio of wav_simulate.py:146-163"""
    if not src_args:
        return None
    paths = src_args.split(",")
    beg_int, end_int = [None] * len(paths), [None] * len(paths)
    if beg:
        beg_int = [int(v) for v in beg.split(",")]
    if end:
        end_int = [int(v) for v in end.split(",")]
    return [read(s, sr=sr, beg=b, end=e) for s, b, e in zip(paths, beg_int, end_int)]


def _select(rir, channel):
    """the RIR selection of add_speaker / add_point_noise (:74-79, :126-131)"""
    rir = np.asarray(rir)
    if rir.ndim == 1:
        rir = rir[None, ...]
    if channel >= 0 and rir.ndim == 2:
        rir = rir[channel:channel + 1]
    if rir.shape[0] == 0:
        raise ValueError(f"--dump-channel {channel} is not a channel of a {rir.ndim}-D RIR")
    return np.ascontiguousarray(rir, dtype=np.float32)


def _room_conv(src, rir, channel):
    """add_room_response (:29-54): ss.convolve(src[None], rir)[..., :S]"""
    if src.ndim != 1:
        raise RuntimeError(f"Can not convolve rir with {src.ndim}D signals")
    return Conv(np.ascontiguousarray(src, dtype=np.float32), _select(rir, channel), src.shape[-1])


def _as2d(a):
    a = np.asarray(a, dtype=np.float32)
    return np.ascontiguousarray(a[None, ...] if a.ndim == 1 else a)


def _slice_len(total, beg, dur):
    """len(range(total)[beg:beg + dur]) -- numpy's slice of a mixture buffer"""
    return len(range(total)[beg:beg + dur])


def plan_mixture(args, name=None, read=read_wav):
    """run_simu (wav_simulate.py:166-312) up to the arithmetic: returns a Mixture, or raises the
    reference's RuntimeError / ValueError."""
    name = name or args.mix
    sr = args.sr

    def arg_float(src_args):
        return [float(s) for s in src_args.split(",")] if src_args else None

    src_spk = _load_audio(args.src_spk, sr=sr, read=read)
    src_rir = _load_audio(args.src_rir, sr=sr, read=read)
    if src_rir:
        if len(src_rir) != len(src_spk):
            raise RuntimeError(f"Number of --src-rir={args.src_rir} do not match with " +
                               f"--src-spk={args.src_spk} option")
    sdr = arg_float(args.src_sdr)
    if len(src_spk) > 1 and not sdr:
        raise RuntimeError("--src-sdr need to be assigned for " + f"--src-spk={args.src_spk}")
    if sdr:
        if len(src_spk) - 1 != len(sdr):
            raise RuntimeError("Number of --src-snr - 1 do not match with " + "--src-snr option")
        sdr = [0] + sdr
    src_begin = arg_float(args.src_begin)
    src_begin = [int(v) for v in src_begin] if src_begin else [0 for _ in src_spk]
    mix_nsamps = max([b + s.size for b, s in zip(src_begin, src_spk)])

    point_noise_rir = _load_audio(args.point_noise_rir, sr=sr, read=read)
    point_noise_end = [str(int(v) + mix_nsamps) for v in args.point_noise_offset.split()]
    point_noise = _load_audio(args.point_noise, beg=args.point_noise_offset, end=",".join(point_noise_end), sr=sr,
                              read=read)
    if args.point_noise:
        if point_noise_rir:
            if len(point_noise) != len(point_noise_rir):
                raise RuntimeError(f"Number of --point-noise-rir={args.point_noise_rir} do not match with " +
                                   f"--point-noise={args.point_noise} option")
        point_snr = arg_float(args.point_noise_snr)
        if not point_snr:
            raise RuntimeError("--point-noise-snr need to be assigned for " + f"--point-noise={args.point_noise}")
        if len(point_noise) != len(point_snr):
            raise RuntimeError(f"Number of --point-noise-snr={args.point_noise_snr} do not match with " +
                               f"--point-noise={args.point_noise} option")
        point_begin = arg_float(args.point_noise_begin)
        point_begin = [int(v) for v in point_begin] if point_begin else [0 for _ in point_noise]

    isotropic_noise = _load_audio(args.isotropic_noise, beg=str(args.isotropic_noise_offset),
                                  end=str(args.isotropic_noise_offset + mix_nsamps), sr=sr, read=read)
    if isotropic_noise:
        isotropic_noise = isotropic_noise[0]
        isotropic_snr = arg_float(args.isotropic_noise_snr)
        if not isotropic_snr:
            raise RuntimeError("--isotropic-snr need to be assigned for " +
                               f"--isotropic-noise={args.isotropic_noise} option")
        isotropic_snr = isotropic_snr[0]

    def bad(what):
        return ValueError(f"{name}: {what}")

    # add_speaker (:57-93)
    ch = args.dump_channel
    mix = Mixture(name, mix_nsamps, 0, float(args.norm_factor))
    for i, spk in enumerate(src_spk):
        if src_rir is None:
            image = _as2d(spk)
        else:
            image = _room_conv(spk, src_rir[i], ch)
        beg = src_begin[i]
        if beg < 0:
            raise bad(f"speaker {i} begins at {beg} < 0")
        mix.terms.append(Term(_lib.SIMU_SPEAKER, image, beg, 0, 0, None, 0.0 if i == 0 else sdr[i]))
    N = mix.terms[0].channels()
    for i, t in enumerate(mix.terms):
        dur = t.samples()
        if t.channels() not in (1, N):
            raise bad(f"could not broadcast speaker {i}'s {t.channels()} channels into {N}")
        t.length, t.power = dur, (0, dur)
    mix.n_channels = N

    # add_point_noise (:96-143)
    if point_noise:
        images, durs = [], []
        for i, noise in enumerate(point_noise):
            beg = point_begin[i]
            if beg < 0 or beg >= mix_nsamps:
                raise bad(f"point noise {i} begins at {beg}, outside [0, {mix_nsamps})")
            if not args.point_noise_repeat:
                dur = min(noise.shape[-1], mix_nsamps - beg)
            else:
                dur = mix_nsamps - beg
                if noise.shape[-1] < dur:
                    noise = np.pad(noise, (0, dur - noise.shape[-1]), mode="wrap")
            if point_noise_rir is None:
                images.append(_as2d(noise))
            else:
                images.append(_room_conv(noise[:dur], point_noise_rir[i], ch))
            durs.append(dur)
        dur = durs[-1]   # the mixing loop's stale `dur`
        n_noise = images[0].h.shape[0] if isinstance(images[0], Conv) else images[0].shape[0]
        for i, image in enumerate(images):
            t = Term(_lib.SIMU_POINT_NOISE, image, point_begin[i], 0, 0, (0, durs[i]), point_snr[i])
            lm, li = _slice_len(mix_nsamps, t.begin, dur), min(t.samples(), dur)
            if t.channels() not in (1, n_noise) or (li != lm and li != 1):
                raise bad(f"could not broadcast point noise {i} of shape ({t.channels()},{li}) into "
                          f"({n_noise},{lm})")
            t.length, t.repeat = lm, int(li != lm)
            mix.terms.append(t)
        if N != n_noise:
            raise RuntimeError("Channel mismatch between source speaker " + "configuration and pointsource noise's, " +
                               f"{N} vs {n_noise}")

    # isotropic noise (:275-302)
    if isotropic_noise is not None:
        iso = isotropic_noise
        if N == 1:
            if iso.ndim == 1:
                iso = iso[None, ...]
            elif ch >= 0:
                iso = iso[ch:ch + 1]
            else:
                raise RuntimeError("Single channel mixture vs multi-channel isotropic noise")
        elif iso.shape[0] != N:
            raise RuntimeError("Channel number mismatch between mixture and isotropic noise, " +
                               f"{N} vs {iso.shape[0]}")
        if iso.ndim != 2 or iso.shape[0] == 0:
            raise IndexError("too many indices for array")
        dur = min(mix_nsamps, iso.shape[-1])
        if dur < 1:
            raise bad("the isotropic noise has no samples at its offset")
        chunk = np.ascontiguousarray(iso[0:1, :dur], dtype=np.float32)
        mix.terms.append(Term(_lib.SIMU_ISOTROPIC, chunk, 0, dur, 0, (0, dur), isotropic_snr))
    return mix


def _image_floats(t):
    if isinstance(t.image, Conv):
        return t.image.h.shape[0] * t.image.n_out
    return int(np.prod(t.image.shape))


def mixture_bytes(m):
    """device bytes one mixture takes in a batch: images, convolution spectra (an estimate) and outputs"""
    img = sum(_image_floats(t) for t in m.terms) * 4
    spec = 0
    for t in m.terms:
        if isinstance(t.image, Conv):
            P = 1024
            spec += 8 * (P + 1) * (-(-t.image.n_out // P) + t.image.h.shape[0] * -(-t.image.h.shape[-1] // P))
            spec += 4 * (t.image.x.shape[-1] + int(np.prod(t.image.h.shape)))
    out = 4 * m.n_samples * (m.n_channels + m.n_speakers() + 1)
    return img + spec + out


def _run_batch(batch, device, pcm16):
    # the pool: every image of the batch, the convolutions' outputs written in place
    offsets, total = [], 0
    for m in batch:
        offs = []
        for t in m.terms:
            offs.append(total)
            total += _image_floats(t)
        offsets.append(offs)
    pool = torch.empty(max(total, 1), dtype=torch.float32, device=device)
    groups = {}
    for mi, m in enumerate(batch):
        for ti, t in enumerate(m.terms):
            if isinstance(t.image, Conv):
                groups.setdefault(t.image.h.shape[0], []).append((mi, ti))
            else:
                img = torch.as_tensor(t.image, dtype=torch.float32).reshape(-1)
                pool[offsets[mi][ti]:offsets[mi][ti] + img.numel()].copy_(img, non_blocking=False)
    for M, items in groups.items():
        convs = [batch[mi].terms[ti].image for mi, ti in items]
        Sx, Lh = max(c.x.shape[-1] for c in convs), max(c.h.shape[-1] for c in convs)
        x = torch.zeros((len(convs), Sx), dtype=torch.float32, device=device)
        h = torch.zeros((len(convs), M, Lh), dtype=torch.float32, device=device)
        for i, c in enumerate(convs):
            x[i, :c.x.shape[-1]] = torch.as_tensor(c.x)
            h[i, :, :c.h.shape[-1]] = torch.as_tensor(c.h)
        s_len = [c.x.shape[-1] for c in convs]
        h_len = [c.h.shape[-1] for c in convs]
        n_out = [c.n_out for c in convs]
        Ny = max(n_out)
        y = torch.empty((len(convs), M, Ny), dtype=torch.float32, device=device)
        plan.convolve(x, h, n_out=n_out, s_len=s_len, h_len=h_len, out=y)
        for i, (mi, ti) in enumerate(items):
            o = offsets[mi][ti]
            pool[o:o + M * n_out[i]].view(M, n_out[i]).copy_(y[i, :, :n_out[i]])
    mixes, terms = [], []
    for mi, m in enumerate(batch):
        mixes.append(dict(first_term=len(terms), n_terms=len(m.terms), n_samples=m.n_samples,
                          n_channels=m.n_channels, norm_factor=m.norm_factor))
        for ti, t in enumerate(m.terms):
            terms.append(dict(src=offsets[mi][ti], kind=t.kind, n_channels=t.channels(), pitch=t.samples(),
                              begin=t.begin, length=t.length, repeat=t.repeat, power_begin=t.power[0],
                              power_end=t.power[1], reserved=0, level_db=float(t.level)))
    M = max(m.n_channels for m in batch)
    K = max(m.n_speakers() for m in batch)
    N = max(m.n_samples for m in batch)
    has_noise = any(t.kind != _lib.SIMU_SPEAKER for m in batch for t in m.terms)
    mix, spk, noise, _ = plan.simulate_mix(pool, mixes, terms, M, K, N, pcm16=pcm16, noise=has_noise)
    mix, spk = mix.cpu(), spk.cpu()
    noise = noise.cpu() if noise is not None else None
    out = []
    for i, m in enumerate(batch):
        T = m.n_samples
        y = mix[i, :m.n_channels, :T].numpy()
        refs = [spk[i, k, :T].numpy() for k in range(m.n_speakers())]
        nz = None
        if any(t.kind != _lib.SIMU_SPEAKER for t in m.terms):
            nz = noise[i, :T].numpy()
        out.append((y[0] if m.n_channels == 1 else y, refs, nz))
    return out


def batches(mixtures, budget=BATCH_BYTES):
    """consecutive groups of mixtures whose device bytes stay within budget (at least one each)"""
    group, used = [], 0
    for m in mixtures:
        b = mixture_bytes(m)
        if group and used + b > budget:
            yield group
            group, used = [], 0
        group.append(m)
        used += b
    if group:
        yield group


def simulate(mixtures, device=None, pcm16=False, budget=BATCH_BYTES):
    """
    Every mixture of `mixtures` (from plan_mixture, or built by hand) on the device, in batches.
    Returns one (mix, [speaker references], noise reference or None) per mixture: mix (N, T), or (T,)
    for one channel; references (T,); float32 or, with pcm16, int16 as write_wav stores them.
    """
    device = torch.device(device if device is not None else ("cuda" if torch.cuda.is_available() else "cpu"))
    out = []
    for group in batches(mixtures, budget):
        out.extend(_run_batch(group, device, pcm16))
    return out


def write_outputs(m, result, dump_ref_dir, sr, write):
    """run()'s file writes (wav_simulate.py:326-341)"""
    mix, spk_ref, noise = result
    write(m.name, mix, sr=sr)
    if dump_ref_dir:
        basename = os.path.basename(m.name)
        ref_dir = os.path.join(dump_ref_dir)
        os.makedirs(ref_dir, exist_ok=True)
        if noise is not None:
            write(os.path.join(ref_dir, "noise", basename), noise, sr=sr)
        if len(spk_ref) == 1:
            write(os.path.join(ref_dir, "clean", basename), spk_ref[0], sr=sr)
        else:
            for i, s in enumerate(spk_ref):
                write(os.path.join(ref_dir, f"spk{i + 1}", basename), s, sr=sr)
