"""
setk_b200.cgmm_cli -- what the CGMM and CACGMM mask estimation command lines behind
scripts/sptk/estimate_cgmm_masks.py and estimate_cacgmm_masks.py share: the loop over the utterances
and the choice of STFT.  Each script keeps its parser, its start, its alignment and its output layout.
"""
from pathlib import Path

import numpy as np
import torch

from .libs.data_handler import NumpyReader, NumpyWriter, ScriptReader, WaveReader
from .libs.utils import default_device, forward_stft, get_logger, get_plan, nextpow2

logger = get_logger(__name__)


class Failed(Exception):
    """An utterance that is logged as "... Failed" and not written; a message, if any, follows in brackets."""


def observe(samps, args, dev):
    """
    samps C x N float32 -> (audio 1 x C x N on dev, plan, stft, T, F).  The tile STFT takes n_fft 512 and
    1024 with a hop that is a multiple of 4: plan is the cached StftPlan and stft None.  Every other
    geometry gets forward_stft per channel: plan None and stft C x F x T complex64.
    """
    C, N = samps.shape
    n_fft = nextpow2(args.frame_len) if args.round_power_of_two else args.frame_len
    audio = torch.from_numpy(np.ascontiguousarray(samps)).to(dev)[None]
    if n_fft in (512, 1024) and args.frame_hop % 4 == 0 and args.frame_hop <= n_fft:
        plan = get_plan(C, args.frame_len, args.frame_hop, bool(args.center), bool(args.round_power_of_two),
                        args.window, N, dev)
        return audio, plan, None, plan.num_frames(N), plan.num_bins
    stft = torch.stack([
        forward_stft(audio[0, c], frame_len=args.frame_len, frame_hop=args.frame_hop,
                     round_power_of_two=bool(args.round_power_of_two), center=bool(args.center),
                     window=args.window, transpose=False) for c in range(C)
    ])
    return audio, None, stft, stft.shape[-1], stft.shape[1]


def run(args, train):
    """
    np.random.seed(args.seed), then train(samps C x N float32, args, init mask or None, device) -> masks
    for every utterance of args.wav_scp whose <args.dst_dir>/<key>.npy does not exist yet, written as
    float32.  The init mask is the entry of args.init_mask (format args.fmt) for the key, if any.
    """
    np.random.seed(args.seed)
    dev = default_device()
    wave_reader = WaveReader(args.wav_scp, sr=16000)
    MaskReader = {"numpy": NumpyReader, "kaldi": ScriptReader}
    init_mask_reader = MaskReader[args.fmt](args.init_mask) if args.init_mask else None

    num_done = 0
    with NumpyWriter(args.dst_dir) as writer:
        dst_dir = Path(args.dst_dir)
        for key, samps in wave_reader:
            if (dst_dir / f"{key}.npy").exists():
                logger.info(f"Training utterance {key} ... Skip")
                continue
            if samps.ndim == 1:
                samps = samps[None]
            init_mask = None
            if init_mask_reader and key in init_mask_reader:
                init_mask = init_mask_reader[key]
            try:
                masks = train(np.asarray(samps, dtype=np.float32), args, init_mask, dev)
            except Failed as err:
                logger.warning(f"Training utterance {key} ... Failed" + (f" ({err})" if err.args else ""))
                continue
            num_done += 1
            writer.write(key, masks.astype(np.float32))
            logger.info(f"Training utterance {key} ... Done")
    logger.info(f"Train {num_done:d} utterances over {len(wave_reader):d}")
