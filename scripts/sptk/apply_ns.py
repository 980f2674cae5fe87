#!/usr/bin/env python
# coding=utf-8
"""
Single channel noise suppression (iMCRA / OM-LSA)

Drop-in for the reference's scripts/sptk/apply_ns.py (same positional arguments, flags and defaults:
StftParser's STFT options, --conf <YAML of iMCRA keywords>, --output {wave,gain}, --sr), with the
STFT, the iMCRA recursion, the inverse STFT and the PCM-16 conversion on libsetk_b200's CUDA kernels
(setk_stft, setk_ns_imcra, setk_istft, setk_float_to_pcm16).
  --output wave  <dst_dir>/<key>.wav: inverse_stft(gain * stft), no peak normalisation, PCM-16
  --output gain  <dst_dir>/<key>.npy: the T x F float64 gain

Kept: --sr other than 16000 raises ValueError, as in the reference.
Repaired reference behaviour: a multichannel input kills the reference's whole run (T, F = stft.shape
raises ValueError on its N x T x F STFT); here that key is logged and skipped, and the run continues.
"""
import argparse
import os
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

import torch  # noqa: E402
import yaml  # noqa: E402

from setk_b200 import plan as _plan  # noqa: E402
from setk_b200.libs.data_handler import NumpyWriter, WaveReader, WaveWriter  # noqa: E402
from setk_b200.libs.ns import iMCRA  # noqa: E402
from setk_b200.libs.opts import StftParser  # noqa: E402
from setk_b200.libs.utils import default_device, get_logger, get_plan  # noqa: E402

logger = get_logger(__name__)


def run(args):
    if args.sr != 16000:
        raise ValueError("Now only support audio in 16kHz")
    if args.conf:
        with open(args.conf, "r") as conf:
            suppressor = iMCRA(**yaml.full_load(conf))
    else:
        suppressor = iMCRA()
    dev = default_device()
    wave_reader = WaveReader(args.wav_scp, sr=args.sr)
    want_wave = args.output == "wave"
    writer = WaveWriter(args.dst_dir, sr=args.sr) if want_wave else NumpyWriter(args.dst_dir)
    num_done = 0
    with writer:
        for key, samps in wave_reader:
            logger.info(f"Processing utterance {key}...")
            if samps.ndim != 1:
                logger.warning(f"{key}: noise suppression needs a single channel input, got "
                               f"{samps.shape[0]} channels; skipped")
                continue
            plan = get_plan(1, args.frame_len, args.frame_hop, bool(args.center), bool(args.round_power_of_two),
                            args.window, samps.shape[-1], dev)
            audio = torch.from_numpy(np.ascontiguousarray(samps, dtype=np.float32)).to(dev)
            stft = plan.stft(audio.reshape(1, 1, -1))[:, 0]                     # 1 x F x T
            gain, enh = _plan.ns_from_stft(stft, config=suppressor.conf, gain=not want_wave, enh=want_wave)
            if want_wave:
                pcm = _plan.float_to_pcm16(plan.istft(enh)[0])
                writer.write(key, pcm.cpu().numpy())
            else:
                writer.write(key, gain[0].cpu().numpy())
            num_done += 1
    logger.info(f"Processed {num_done:d} utterances over {len(wave_reader):d}")


if __name__ == "__main__":
    parser = argparse.ArgumentParser(
        description="Command to do single channel noise suppression",
        formatter_class=argparse.ArgumentDefaultsHelpFormatter,
        parents=[StftParser.parser])
    parser.add_argument("wav_scp", type=str, help="Noisy audio scripts in Kaldi format")
    parser.add_argument("dst_dir", type=str, help="Location to dump enhanced audio or gain coefficients")
    parser.add_argument("--conf", type=str, default="", help="Yaml configurations for OMLSA")
    parser.add_argument("--output", type=str, choices=["gain", "wave"], default="wave",
                        help="Output type of the command")
    parser.add_argument("--sr", type=int, default=16000, help="Waveform data sample frequency")
    args = parser.parse_args()
    run(args)
