"""
setk_b200.cli_tools -- the feature / WPD command lines behind scripts/sptk/
{compute_ipd_and_linear_srp, compute_df_on_geometry, compute_circular_srp, apply_wpd}.py.

Each keeps the positional arguments, flag names, destinations and defaults of the reference
script of the same name (scripts/sptk/*.py of funcwj/setk; cited per function) so that recipes
written against the reference keep working; everything numeric runs on libsetk_b200's CUDA
kernels through setk_b200.libs.  Flags are declared as tables (name, type, default, dest, help).
"""
import argparse

import numpy as np
import torch

from .libs.data_handler import ArchiveWriter, ScpReader, SpectrogramReader, WaveWriter
from .libs.opts import StftParser, str2tuple, strtobool
from .libs.utils import get_logger, inverse_stft, nextpow2

logger = get_logger(__name__)


def _parser(description, positionals, flags):
    p = argparse.ArgumentParser(description=description,
                                formatter_class=argparse.ArgumentDefaultsHelpFormatter,
                                parents=[StftParser.parser])
    for name, text in positionals:
        p.add_argument(name, type=str, help=text)
    for name, typ, default, dest, text in flags:
        kw = dict(type=typ, default=default, help=text)
        if dest:
            kw["dest"] = dest
        p.add_argument(name, **kw)
    return p


def _stft_options(args, transpose):
    return dict(frame_len=args.frame_len, frame_hop=args.frame_hop, window=args.window,
                center=args.center, round_power_of_two=args.round_power_of_two, transpose=transpose)


def _bins(args):
    n = nextpow2(args.frame_len) if args.round_power_of_two else args.frame_len
    return n // 2 + 1


def _pairs(text, flag):
    pairs = []
    for item in text.split(";"):
        idx = [int(v) for v in item.split(",")]
        if len(idx) != 2:
            raise ValueError(f"Invalid {flag} configuration detected: {text}")
        pairs.append(tuple(idx))
    if not pairs:
        raise RuntimeError(f"Bad configurations with {flag} {text}")
    return pairs


def _each_stft(reader):
    """(key, samples, STFT as a device tensor) for every utterance of a SpectrogramReader."""
    for key in reader.index_keys:
        samps = reader.read(key)
        yield key, samps, reader.stft(samps, as_tensor=True)


def _dump_archive(args_ark, args_scp, items, what):
    done = 0
    with ArchiveWriter(args_ark, args_scp) as writer:
        for key, feats in items:
            writer.write(key, feats.cpu().numpy())
            done += 1
            if done % 1000 == 0:
                logger.info(f"Processed {done} utterances...")
    logger.info(f"Processed {what} for {done} utterances")


# ---------------------------------------------------------------------------------------------
# compute_ipd_and_linear_srp.py (reference: compute_spatial_feats :21-50, run :53-73, flags :76-143)
# ---------------------------------------------------------------------------------------------
def spatial_feats_main(argv=None):
    from .libs.spatial import ipd, msc, srp_phat_linear
    args = _parser(
        "Spatial features of a multi-channel recording: SRP-PHAT angular spectrum of a linear array "
        "(srp), magnitude squared coherence (msc) or inter-channel phase differences (ipd)",
        [("wav_scp", "multi-channel wave script (Kaldi format)"),
         ("dup_ark", "Kaldi archive the features are written to")],
        [("--scp", str, "", None, "also write the archive's script file here"),
         ("--type", str, "srp", None, "srp | msc | ipd"),
         ("--srp.sample-rate", int, 16000, "samp_frequency", "sample rate of the input"),
         ("--srp.sample-tdoa", strtobool, False, "samp_tdoa", "sample the TDoA axis instead of the DoA axis"),
         ("--srp.num_doa", int, 181, "num_doa", "directions sampled between 0 and 180 degrees"),
         ("--srp.topo", str2tuple, "0,0.2,0.4,0.8", "linear_topo", "microphone positions of the linear array"),
         ("--ipd.cos", strtobool, False, "ipd_cos", "cosIPD instead of IPD"),
         ("--ipd.sin", strtobool, False, "ipd_sin", "append sinIPD to cosIPD"),
         ("--ipd.pair", str, "0,1", "ipd_pair", "channel pairs, e.g. 0,3;1,4"),
         ("--msc.ctx", int, 1, "msc_ctx", "frame context of the coherence estimate")]).parse_args(argv)
    if args.type not in ("srp", "msc", "ipd"):
        raise SystemExit(f"--type: invalid choice {args.type!r}")

    def features(S):                                   # S: N x T x F on the device
        if args.type == "srp":
            return srp_phat_linear(S, args.linear_topo, sample_frequency=args.samp_frequency,
                                   num_doa=args.num_doa, num_bins=_bins(args), samp_doa=not args.samp_tdoa)
        if args.type == "msc":
            return msc(S, context=args.msc_ctx)
        if S.ndim < 3:
            raise ValueError("Only one-channel STFT available")
        cols = []
        for left, right in _pairs(args.ipd_pair, "--ipd.pair"):
            if right > S.shape[0]:
                raise RuntimeError(f"Could not access channel {right}")
            cols.append(ipd(S[left], S[right], cos=args.ipd_cos, sin=args.ipd_sin))
        return torch.cat(cols, dim=1)

    reader = SpectrogramReader(args.wav_scp, **_stft_options(args, transpose=True))
    _dump_archive(args.dup_ark, args.scp, ((k, features(S)) for k, _, S in _each_stft(reader)),
                  args.type.upper())


# ---------------------------------------------------------------------------------------------
# compute_df_on_geometry.py (reference: run :18-71, flags :74-112)
# ---------------------------------------------------------------------------------------------
def df_on_geometry_main(argv=None):
    from .libs.spatial import directional_feats
    args = _parser(
        "Directional features of a linear array for given steering vectors",
        [("wav_scp", "multi-channel wave script (Kaldi format)"),
         ("steer_vector", "steering vectors, .npy of shape A x M x F (directions x microphones x bins)"),
         ("dup_ark", "Kaldi archive the features are written to")],
        [("--utt2idx", str, "", None, "per-utterance direction index in [0, A - 1]"),
         ("--doa-idx", str, 0, None, "direction index (or comma list) for all utterances without --utt2idx"),
         ("--scp", str, "", None, "also write the archive's script file here"),
         ("--df-pair", str, "0,1", None, "microphone pairs, e.g. 0,1;0,2")]).parse_args(argv)
    pairs = _pairs(args.df_pair, "--df-pair")
    table = np.load(args.steer_vector)
    utt2idx = ScpReader(args.utt2idx, value_processor=int) if args.utt2idx else None
    logger.info(f"Compute directional feature with {pairs}")

    def items():
        reader = SpectrogramReader(args.wav_scp, **_stft_options(args, transpose=False))
        for key, _, S in _each_stft(reader):           # S: M x F x T
            if utt2idx is not None:
                if key not in utt2idx:
                    logger.warning(f"Missing utt2idx for utterance {key}")
                    continue
                yield key, directional_feats(S, table[utt2idx[key]], df_pair=pairs)
                continue
            chosen = [int(v) for v in str(args.doa_idx).split(",")]
            per_dir = [directional_feats(S, table[i], df_pair=pairs) for i in chosen]
            if len(per_dir) == 1:
                yield key, per_dir[0]
            else:                                       # T x (directions * F)
                stacked = torch.stack(per_dir)
                yield key, stacked.transpose(0, 1).reshape(stacked.shape[1], -1)

    _dump_archive(args.dup_ark, args.scp, items(), "DF")


# ---------------------------------------------------------------------------------------------
# compute_circular_srp.py (reference: run :17-58, flags :61-92)
# ---------------------------------------------------------------------------------------------
def circular_srp_main(argv=None):
    from .libs.spatial import gcc_phat_diag
    args = _parser(
        "SRP angular spectrum of a circular array from its diagonal microphone pairs",
        [("wav_scp", "multi-channel wave script (Kaldi format)"),
         ("srp_ark", "Kaldi archive the spectra are written to")],
        [("--scp", str, "", None, "also write the archive's script file here"),
         ("--n", int, 6, None, "microphones on the circle"),
         ("--d", float, 0.07, None, "diameter of the array in metres"),
         ("--diag-pair", str, "0,3;1,4;2,5", None, "diagonal pairs whose GCC-PHAT is averaged"),
         ("--sr", int, 16000, None, "sample rate of the input"),
         ("--num-doas", int, 121, None, "directions sampled between 0 and 2 pi")]).parse_args(argv)
    pairs = _pairs(args.diag_pair, "--diag-pair")
    logger.info(f"Compute gcc with {pairs}")

    def items():
        reader = SpectrogramReader(args.wav_scp, **_stft_options(args, transpose=True))
        for key, _, S in _each_stft(reader):           # S: N x T x F
            acc = None
            for i, j in pairs:
                g = gcc_phat_diag(S[i], S[j], min(i, j) * np.pi * 2 / args.n, args.d, num_bins=_bins(args),
                                  sr=args.sr, num_doas=args.num_doas)
                acc = g if acc is None else acc + g
            srp = acc / len(pairs)
            bad = int(torch.isnan(srp).sum())
            if bad:
                raise RuntimeError(f"Matrix {key} has nan ({bad:d}) items)")
            yield key, srp

    _dump_archive(args.srp_ark, args.scp, items(), "SRP")


# ---------------------------------------------------------------------------------------------
# apply_wpd.py (reference: run :20-59, flags :62-109)
# ---------------------------------------------------------------------------------------------
def wpd_main(argv=None):
    from .libs.wpe import facted_wpd
    args = _parser(
        "Joint dereverberation and denoising with the factored WPD beamformer",
        [("wav_scp", "multi-channel wave script (Kaldi format)"),
         ("dst_dir", "directory the enhanced audio is written to")],
        [("--taps", int, 10, None, "prediction taps of the WPE stage"),
         ("--delay", int, 3, None, "prediction delay of the WPE stage"),
         ("--context", int, 1, None, "frame context of the first variance estimate"),
         ("--wpd-iters", int, 3, None, "WPD iterations"),
         ("--cgmm-iters", int, 20, None, "CGMM iterations inside every WPD iteration"),
         ("--update-alpha", strtobool, False, None, "update the CGMM priors in the M-step"),
         ("--sr", int, 16000, None, "sample rate of the input"),
         ("--dump-mask", strtobool, False, None, "also save the speech mask as <dst_dir>/<key>.npy")]
    ).parse_args(argv)
    opts = _stft_options(args, transpose=True)
    reader = SpectrogramReader(args.wav_scp, **opts)
    opts.pop("round_power_of_two")
    done = 0
    with WaveWriter(args.dst_dir, sr=args.sr) as writer:
        for key, samps, obs in _each_stft(reader):      # obs: N x T x F
            logger.info(f"Processing utt {key}...")
            if obs.ndim != 3:
                raise RuntimeError(f"Expected 3D array, but got {obs.ndim}")
            try:
                tf_mask, enh = facted_wpd(obs, wpd_iters=args.wpd_iters, cgmm_iters=args.cgmm_iters,
                                          update_alpha=args.update_alpha, context=args.context,
                                          taps=args.taps, delay=args.delay)
            except np.linalg.LinAlgError:
                logger.warning(f"{key}: Failed cause LinAlgError in wpd")
                continue
            wave = inverse_stft(enh, norm=float(np.max(np.abs(samps))), **opts)
            writer.write(key, wave.cpu().numpy())
            if args.dump_mask:
                np.save(f"{args.dst_dir}/{key}", tf_mask[..., 0].cpu().numpy())
            done += 1
            if done % 100 == 0:
                logger.info(f"Processed {done:d} utterances...")
    logger.info(f"Processed {done:d} utterances over {len(reader):d}")


# ---------------------------------------------------------------------------------------------
# compute_df_on_mask.py (reference: run :21-59, flags :62-95)
# ---------------------------------------------------------------------------------------------
def df_on_mask_main(argv=None):
    from .libs.beamformer import compute_covar, solve_pevd
    from .libs.data_handler import NumpyReader, ScriptReader
    from .libs.spatial import directional_feats
    args = _parser(
        "Directional features of an arbitrary array; the steering vector is the principal eigenvector "
        "of the mask-weighted spatial covariance",
        [("wav_scp", "multi-channel wave script (Kaldi format)"),
         ("mask_scp", "script of the TF-masks (Kaldi archive entries or .npy files)"),
         ("dup_ark", "Kaldi archive the features are written to")],
        [("--scp", str, "", None, "also write the archive's script file here"),
         ("--mask-format", str, "kaldi", "fmt", "kaldi | numpy"),
         ("--df-pair", str, "0,1", None, "microphone pairs, e.g. 0,1;0,2")]).parse_args(argv)
    if args.fmt not in ("kaldi", "numpy"):
        raise SystemExit(f"--mask-format: invalid choice {args.fmt!r}")
    pairs = _pairs(args.df_pair, "--df-pair")
    masks = (NumpyReader if args.fmt == "numpy" else ScriptReader)(args.mask_scp)
    logger.info(f"Compute directional feature with {pairs}")

    def items():
        reader = SpectrogramReader(args.wav_scp, **_stft_options(args, transpose=False))
        for key, _, obs in _each_stft(reader):          # obs: N x F x T
            if key not in masks:
                logger.warning(f"Missing TF-mask for utterance {key}")
                continue
            m = masks[key]
            if m.shape[0] == obs.shape[1]:              # given as F x T
                m = np.transpose(m)
            m = torch.from_numpy(np.ascontiguousarray(np.minimum(m, 1)))
            steer = solve_pevd(compute_covar(obs, m))   # F x N
            yield key, directional_feats(obs, steer.transpose(0, 1), df_pair=pairs)

    _dump_archive(args.dup_ark, args.scp, items(), "DF")


# ---------------------------------------------------------------------------------------------
# do_ssl.py (reference: add_wta :17-27, get_doa :30-37, run :40-115, flags :118-172)
# ---------------------------------------------------------------------------------------------
def add_wta(masks_list, eps=1e-4):
    """Winner-take-all masks (do_ssl.py:17-27): a cell keeps its value where it is the largest."""
    top = np.max(np.stack(masks_list, axis=-1), -1)
    return [np.where(m == top, m, eps) for m in masks_list]


def ssl_windows(T, chunk_len, look_back):
    """
    Frame windows of do_ssl.py: [0, T) offline; online (chunk_len > 0 and look_back > 0) the chunks
    [max(t - look_back, 0), min(t + chunk_len, T)) for t = 0, chunk_len, ... (:63,103-109).
    """
    if chunk_len > 0 and look_back > 0:
        return [(max(t - look_back, 0), min(t + chunk_len, T)) for t in range(0, T, chunk_len)]
    return [(0, T)]


def ssl_main(argv=None):
    """
    Sound source localisation with ML / SRP / MUSIC, optionally informed by TF-masks.

    One deliberate difference from the reference: in online mode with a mask, do_ssl.py:106
    slices mask[..., s:t + chunk_len] after the mask has become T x F, i.e. it cuts FREQUENCY
    bins, and ml_ssl then fails with a broadcast ValueError.  Here every chunk uses the mask's
    frames s .. t + chunk_len - 1, the same frames as its STFT chunk.
    """
    from . import plan as _plan
    from .libs.data_handler import NumpyReader
    from .libs.utils import EPSILON, default_device
    args = _parser(
        "Command to ML/SRP based sound souce localization (SSL).Also see scripts/sptk/compute_steer_vector.py",
        [("wav_scp", "Multi-channel wave rspecifier"),
         ("steer_vector", "Pre-computed steer vector in each directions (in shape A x M x F, A: number of "
                          "DoAs, M: microphone number, F: FFT bins)"),
         ("doa_scp", "Wspecifier for estimated DoA")],
        [("--backend", str, "ml", None, "Which algorithm to choose for SSL (ml | srp | music)"),
         ("--srp-pair", str, "", None, "Microphone index pair to compute srp response"),
         ("--doa-range", str, "0,360", None, "DoA range"),
         ("--mask-scp", str, "", None, "Rspecifier for TF-masks in numpy format"),
         ("--output", str, "degree", None, "Output type of the DoA (radian | degree | index)"),
         ("--mask-eps", float, -1, None, "Value of eps used in masking winner-take-all"),
         ("--chunk-len", int, -1, None, "Number frames per chunk (for online setups)"),
         ("--look-back", int, 125, None, "Number of frames to look back (for online setups)")]).parse_args(argv)
    if args.backend not in ("ml", "srp", "music"):
        raise SystemExit(f"--backend: invalid choice {args.backend!r}")
    if args.output not in ("radian", "degree", "index"):
        raise SystemExit(f"--output: invalid choice {args.output!r}")
    steer_vector = np.load(args.steer_vector)
    logger.info(f"Shape of the steer vector: {steer_vector.shape}")
    num_doa = steer_vector.shape[0]
    min_doa, max_doa = str2tuple(args.doa_range)
    if args.output == "radian":
        angles = np.linspace(min_doa * np.pi / 180, max_doa * np.pi / 180, num_doa + 1)
    else:
        angles = np.linspace(min_doa, max_doa, num_doa + 1)
    reader = SpectrogramReader(args.wav_scp, **_stft_options(args, transpose=False))
    mask_reader = [NumpyReader(scp) for scp in args.mask_scp.split(",")] if args.mask_scp else None
    online = args.chunk_len > 0 and args.look_back > 0
    if online:
        logger.info(f"Set up in online mode: chunk_len = {args.chunk_len}, look_back = {args.look_back}")
    pairs = None
    if args.backend == "srp":
        pairs = _pairs(args.srp_pair, "--srp-pair")
        logger.info(f"Choose srp-based algorithm, srp pair is "
                    f"{([p[0] for p in pairs], [p[1] for p in pairs])}")
    steer = torch.as_tensor(steer_vector, device=default_device()).to(torch.complex128)
    kw = dict(compression=-1, eps=EPSILON) if args.backend == "ml" else {}

    def label(i):
        return float(i) if args.output == "index" else angles[i]

    done = 0
    with open(args.doa_scp, "w") as doa_out:
        for key, _, S in _each_stft(reader):               # S: M x F x T on the device
            _, F, T = S.shape
            mask = None
            if mask_reader:
                mask = [r[key] for r in mask_reader]
                if args.mask_eps >= 0 and len(mask_reader) > 1:
                    mask = add_wta(mask, eps=args.mask_eps)
                mask = mask[0]
                if mask.shape[-1] != F:                     # F x T => T x F
                    mask = mask.transpose()
                mask = torch.from_numpy(np.ascontiguousarray(mask, dtype=np.float32))[None, None]
            windows = ssl_windows(T, args.chunk_len, args.look_back)
            _, index = _plan.ssl(S[None], steer, backend=args.backend, mask=mask, windows=[windows],
                                 pairs=pairs, **kw)
            doa = [label(i) for i in index[0, 0].cpu().tolist()]
            if not online:
                logger.info(f"Processing utterance {key}: {doa[0]:.4f}")
                doa_out.write(f"{key}\t{doa[0]:.4f}\n")
            else:
                logger.info(f"Processing utterance {key}...")
                doa_out.write(f"{key}\t" + " ".join(f"{d:.4f}" for d in doa) + "\n")
            done += 1
    logger.info(f"Processing {done} utterance done")


# ---------------------------------------------------------------------------------------------
# compute_steer_vector.py (reference: run :17-51, flags :54-105)
# ---------------------------------------------------------------------------------------------
def steer_vector_main(argv=None):
    """
    Steering vectors A x M x F (complex128 .npy) of a linear or circular array.  Geometry
    constants computed on the host with numpy, like the fixed beamformers' weights.
    """
    from .libs.beamformer import circular_steer_vector, linear_steer_vector
    p = argparse.ArgumentParser(description="Command to compute steer vectors, using for SSL & BF & AF computation",
                                formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument("steer_vector", type=str, help="Output location of the steer vector")
    for name, typ, default, text in (
            ("--num-doas", int, 181, "Step size when sampling the DoA"),
            ("--num-bins", int, 257, "Number of the FFT points used"),
            ("--sr", int, 16000, "Sample rate of input wave"),
            ("--speed", float, 343, "Speed of sound"),
            ("--linear-topo", str2tuple, (), "Topology of linear microphone arrays"),
            ("--circular-around", int, 6, "Number of the micriphones in circular arrays"),
            ("--circular-radius", float, 0.05, "Radius of circular array"),
            ("--circular-center", strtobool, False, "Is there a microphone put in the center of the circular array?"),
            ("--geometry", str, "linear", "Geometry of the microphone array (linear | circular)"),
            ("--normalize", strtobool, False, "Normalzed steer vector or not")):
        p.add_argument(name, type=typ, default=default, help=text)
    args = p.parse_args(argv)
    if args.geometry not in ("linear", "circular"):
        raise SystemExit(f"--geometry: invalid choice {args.geometry!r}")
    if args.geometry == "linear":
        topo = np.array(args.linear_topo)
        candidate_doa = np.linspace(0, 180, args.num_doas)
        sv = [linear_steer_vector(topo, doa, args.num_bins, c=args.speed, sr=args.sr) for doa in candidate_doa]
    else:
        candidate_doa = np.arange(0, 360, 360 / args.num_doas)
        sv = [circular_steer_vector(args.circular_radius, args.circular_around, doa, args.num_bins, c=args.speed,
                                    sr=args.sr, center=args.circular_center) for doa in candidate_doa]
    sv = np.stack(sv)                                       # A x F x M
    if args.normalize:
        sv = sv / sv.shape[-1]**0.5
    np.save(args.steer_vector, sv.transpose(0, 2, 1))       # A x M x F


# ---------------------------------------------------------------------------------------------
# compute_spectrogram.py (reference: run :19-40, flags :43-84) and compute_fbank.py (run :22-61,
# flags :64-121): ragged device batches of channel 0.  A reader thread loads consecutive keys (raw
# int16 for PCM-16 files); two pinned staging sets alternate, so that filling one overlaps the device
# work and the copy back of the other; H2D, setk_pcm16_to_float, setk_spectral_feats, D2H; entries are
# written in scp order.  The bytes written do not depend on --batch-size.
# ---------------------------------------------------------------------------------------------
_FEAT_FORMATS = ("kaldi", "exraw")
_FEAT_FLAGS = [("--scp", str, "", None, "If assigned, generate corresponding scripts for archives"),
               ("--format", str, "kaldi", None, "Output archive format (kaldi | exraw), see sptk/libs/exraw.py"),
               ("--batch-size", int, 64, "batch_size", "utterances per device batch")]


class _FeatStaging(object):
    """One pinned host set: int16 or float32 input [B][N], lengths, features out [B][T][D], and its event."""

    def __init__(self, batch, n_cap, t_cap, D, pcm16, pin):
        self.pcm16 = pcm16
        self.x = torch.zeros((batch, n_cap), dtype=torch.int16 if pcm16 else torch.float32, pin_memory=pin)
        self.lens = torch.zeros((batch,), dtype=torch.int32, pin_memory=pin)
        self.out = torch.empty((batch, t_cap, D), dtype=torch.float32, pin_memory=pin)
        self.event = None
        self.job = None


def _feature_batches(reader, batch_size):
    """Lists of (key, channel-0 samples) of consecutive keys, loaded by a background thread."""
    import queue
    import threading
    q = queue.Queue(maxsize=4)
    err = []

    def load():
        try:
            batch = []
            for key in reader.index_keys:
                x = reader.read(key)
                batch.append((key, np.ascontiguousarray(x[0] if x.ndim == 2 else x)))
                if len(batch) == batch_size:
                    q.put(batch)
                    batch = []
            if batch:
                q.put(batch)
        except BaseException as e:     # surfaced by the consumer
            err.append(e)
        finally:
            q.put(None)

    threading.Thread(target=load, daemon=True).start()
    while True:
        batch = q.get()
        if batch is None:
            break
        yield batch
    if err:
        raise err[0]


def _run_features(args, apply_log, apply_pow=False, mel_args=None, normalize=True):
    """
    Features of channel 0 of every utterance of args.wav_scp.  normalize=False feeds the raw sample
    values (read_wav(normalize=False): int16 values of PCM-16, data >> 16 of 32-bit PCM, ...).  Every
    utterance is staged as its normalised-domain samples v = raw / 32768 (PCM-16 on the device, other
    formats on the host, exactly: a power of two) and setk_spectral_feats scales |X| back by 32768, so
    an utterance gives the same bits whatever else shares its batch.
    """
    from . import plan as _plan
    from .libs.exraw import BinaryWriter
    from .libs.utils import default_device, get_plan
    from .libs.data_handler import WaveReader
    if args.format not in _FEAT_FORMATS:
        raise SystemExit(f"--format: invalid choice {args.format!r}")
    if args.batch_size < 1:
        raise SystemExit("--batch-size must be >= 1")
    dev = default_device()
    reader = WaveReader(args.wav_scp, normalize=normalize, raw_pcm16=True)
    sample_scale = 1.0 if normalize else 32768.0
    writer_cls = ArchiveWriter if args.format == "kaldi" else BinaryWriter
    D = mel_args["n_mels"] if mel_args else _bins(args)
    weights = None
    if mel_args:
        from .libs.filters import mel
        n_fft = nextpow2(args.frame_len) if args.round_power_of_two else args.frame_len
        weights = mel(args.sr, n_fft, htk=True, **mel_args)
    staging = [None, None]
    mel_plan = [None]
    done = [0]

    def finish(writer, st):
        st.event.synchronize()
        for b, (key, T) in enumerate(st.job):
            writer.write(key, st.out[b, :T].numpy().copy())
            done[0] += 1
        st.job = None

    def host_samples(x):
        """x in the normalised domain as float32 (exact: x / 32768 or x as read)."""
        if x.dtype == np.int16 or not normalize:
            return x.astype(np.float32) / np.float32(32768.0)
        return x.astype(np.float32)

    short = None     # the error of an utterance too short for one frame, raised once the keys before it are written
    with writer_cls(args.dup_ark, args.scp) as writer:
        try:
            for i, batch in enumerate(_feature_batches(reader, args.batch_size)):
                N = max(x.shape[-1] for _, x in batch)
                pl = get_plan(1, args.frame_len, args.frame_hop, args.center, args.round_power_of_two, args.window,
                              N, dev, batch=args.batch_size)
                frames = []
                for j, (_, x) in enumerate(batch):
                    try:
                        frames.append(pl.num_frames(x.shape[-1]))
                    except ValueError as e:          # librosa's error on a too-short input stops the run
                        short, batch = e, batch[:j]
                        break
                if batch:
                    B = len(batch)
                    N = max(x.shape[-1] for _, x in batch)
                    T = pl.num_frames(N)
                    pcm16 = all(x.dtype == np.int16 for _, x in batch)
                    if weights is not None and mel_plan[0] is not pl:
                        pl.set_mel(weights)
                        mel_plan[0] = pl
                    st = staging[i % 2]
                    if st is not None and st.job is not None:
                        finish(writer, st)
                    if st is None or st.pcm16 != pcm16 or st.x.shape[1] < N or st.out.shape[1] < T:
                        st = staging[i % 2] = _FeatStaging(args.batch_size, N, T, D, pcm16, dev.type == "cuda")
                    xs = st.x[:B, :N]
                    xs.zero_()
                    for b, (_, x) in enumerate(batch):
                        xs[b, :x.shape[-1]] = torch.from_numpy(x if pcm16 else host_samples(x))
                        st.lens[b] = x.shape[-1]
                    x_dev = xs.to(dev, non_blocking=True)
                    audio = (_plan.pcm16_to_float(x_dev) if pcm16 else x_dev).view(B, 1, N)
                    lens = st.lens[:B].to(dev, non_blocking=True)
                    feats = pl.spectral_feats(audio, n_samples=lens, apply_pow=apply_pow, mel=weights is not None,
                                              apply_log=apply_log, sample_scale=sample_scale)
                    st.out[:B, :T].copy_(feats[:, 0], non_blocking=True)
                    if dev.type == "cuda":
                        st.event = torch.cuda.Event()
                        st.event.record(torch.cuda.current_stream(dev))
                    else:
                        st.event = type("_Done", (), {"synchronize": staticmethod(lambda: None)})
                    st.job = [(key, t) for (key, _), t in zip(batch, frames)]
                    if done[0] and done[0] % 1000 < B:
                        logger.info(f"Processed {done[0]} utterances...")
                    prev = staging[(i + 1) % 2]
                    if prev is not None and prev.job is not None:
                        finish(writer, prev)
                if short is not None:
                    break
        finally:    # the keys before a failure are written, as the reference's loop writes them
            for st in staging:      # each batch finishes the one before it: at most one is pending here
                if st is not None and st.job is not None:
                    finish(writer, st)
    if short is not None:
        raise short
    logger.info("Process {:d} utterances".format(done[0]))


def spectrogram_main(argv=None):
    args = _parser(
        "Command to extract spectrogram features (magnitude, power or log, channel 0) on the GPU and write "
        "them as Kaldi (or exraw) archives",
        [("wav_scp", "Source location of wave scripts in kaldi format"),
         ("dup_ark", "Location to dump spectrogram features")],
        _FEAT_FLAGS + [
            ("--apply-log", strtobool, False, None, "If true, using log spectrogram instead of linear"),
            ("--apply-pow", strtobool, False, None, "If true, extract power spectrum instead of magnitude spectrum"),
            # parsed and never passed on by the reference: samples are always int16 / 32768
            ("--normalize-samples", strtobool, False, "normalize", "If true, normalize sample values between "
             "[-1, 1] (accepted and ignored, as in the reference)")]).parse_args(argv)
    _run_features(args, args.apply_log, apply_pow=args.apply_pow)


def fbank_main(argv=None):
    args = _parser(
        "Command to extract mel-spectrogram/fbank features (channel 0) on the GPU and write them as Kaldi "
        "(or exraw) archives",
        [("wav_scp", "Source location of wave scripts in kaldi format"),
         ("dup_ark", "Location to dump spectrogram's features")],
        _FEAT_FLAGS + [
            ("--sr", int, 16000, None, "Waveform data sample rate"),
            ("--apply-log", strtobool, False, "log", "If true, using log mel-spectrogram instead of linear"),
            ("--normalize-samples", strtobool, False, "norm", "If true, normalize sample values between [-1, 1]"),
            ("--num-bins", int, 40, "num_bins", "Number of mel-bins defined in mel-filters"),
            ("--min-freq", int, 0, "min_freq", "Low cutoff frequency for mel bins"),
            ("--max-freq", int, 8000, "max_freq", "High cutoff frequency for mel bins")]).parse_args(argv)
    if args.max_freq > args.sr // 2:
        raise RuntimeError("Max frequency for mel exceeds sample frequency")
    _run_features(args, args.log, mel_args=dict(n_mels=args.num_bins, fmin=args.min_freq, fmax=args.max_freq),
                  normalize=args.norm)
