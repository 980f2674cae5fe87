#!/usr/bin/env python
# coding=utf-8
"""
AuxIVA blind source separation

Drop-in for the reference's scripts/sptk/apply_auxiva.py (same positional arguments, flags,
defaults and outputs: <dst_dir>/<key>.src{1..N}.wav, PCM-16, each source peak-normalised to the
input's max |sample|), with the STFT, the AuxIVA epochs and the inverse STFT on libsetk_b200's CUDA
kernels (setk_stft, setk_auxiva_stft, setk_istft).  auxiva(X, epochs) keeps the reference's
signature: N x T x F in, N x T x F complex128 out.

Repaired reference behaviour: the reference lets numpy.linalg.LinAlgError escape when W^H V is
exactly singular (an all-zero bin, a silent channel) and the whole run dies; here that utterance is
logged and skipped, and the run continues.
"""
import argparse
import os
import sys
from pathlib import Path

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

import torch  # noqa: E402

from setk_b200 import plan as _plan  # noqa: E402
from setk_b200.libs.data_handler import WaveReader  # noqa: E402
from setk_b200.libs.opts import StftParser  # noqa: E402
from setk_b200.libs.utils import default_device, get_logger, get_plan, write_wav  # noqa: E402

logger = get_logger(__name__)


def _separate(stft, epochs):
    """stft (N, F, T) complex64 tensor -> (N, F, T) complex128; LinAlgError like the reference."""
    Y, status = _plan.auxiva_from_stft(stft[None], num_epochs=epochs)
    if int(status[0]):
        raise np.linalg.LinAlgError("Singular matrix")
    return Y[0]


def auxiva(X, epochs=20):
    """
    Arguments:
        X: shape in N x T x F
    Return
        Y: same shape as X (complex128)
    """
    x = torch.as_tensor(np.ascontiguousarray(np.transpose(X, (0, 2, 1)))).to(default_device())
    return np.ascontiguousarray(np.transpose(_separate(x, epochs).cpu().numpy(), (0, 2, 1)))


def run(args):
    dev = default_device()
    wave_reader = WaveReader(args.wav_scp)
    num_done = 0
    for key, samps in wave_reader:
        logger.info(f"Processing utterance {key}...")
        if samps.ndim == 1:
            raise RuntimeError(f"{key}: AuxIVA needs a multi-channel input")
        N, S = samps.shape
        plan = get_plan(N, args.frame_len, args.frame_hop, bool(args.center), bool(args.round_power_of_two),
                        args.window, S, dev, batch=N)
        audio = torch.from_numpy(np.ascontiguousarray(samps, dtype=np.float32)).to(dev)[None]
        try:
            separated = _separate(plan.stft(audio)[0], args.epochs)             # N x F x T
        except np.linalg.LinAlgError:
            logger.warning(f"{key}: Failed cause LinAlgError in auxiva")
            continue
        norm = np.max(np.abs(samps))
        # every source is one "utterance" of the inverse STFT, peak-normalised when norm != 0
        out = plan.istft(separated.to(torch.complex64), norm=[norm] * N if norm else None).cpu().numpy()
        for idx in range(N):
            write_wav(Path(args.dst_dir) / f"{key}.src{idx + 1}.wav", out[idx], sr=args.sr)
        num_done += 1
    logger.info(f"Processed {num_done:d} utterances over {len(wave_reader):d}")


if __name__ == "__main__":
    parser = argparse.ArgumentParser(
        description="Command to do AuxIVA bss algorithm",
        formatter_class=argparse.ArgumentDefaultsHelpFormatter,
        parents=[StftParser.parser])
    parser.add_argument("wav_scp", type=str, help="Multi-channel wave scripts in kaldi format")
    parser.add_argument("dst_dir", type=str, help="Location to dump separated source files")
    parser.add_argument("--num-epochs", default=20, type=int, dest="epochs",
                        help="Number of epochs to run AuxIVA algorithm")
    parser.add_argument("--sr", type=int, default=16000, help="Waveform data sample rate")
    args = parser.parse_args()
    run(args)
