#!/usr/bin/env python
# coding=utf-8
"""
Speaker masks estimation with a complex angular central Gaussian mixture model (CACGMM)

Drop-in for the reference's scripts/sptk/estimate_cacgmm_masks.py (same positional arguments,
flags, defaults and outputs: <dst_dir>/<key>.npy, float32 K x T x F for every K; utterances whose
.npy exists are skipped and draw no random numbers), with the STFT, the EM iterations and the
permutation alignment on libsetk_b200's CUDA kernels (setk_cacgmm_masks: tile STFT into a
bin-major workspace, fp64 covariance / eigen / posterior kernels on the unit-norm observations,
then the aligner on the fp64 posteriors; csrc/cgmm.cu, csrc/permu.cu).  Frame sizes other than
512 / 1024 points go through the generic STFT and setk_cacgmm_stft.

Notes against the reference:
  * the random start is drawn with numpy after np.random.seed(--seed), once per trained
    utterance in file order, as the reference's CacgmmTrainer draws it, and handed to the GPU in
    float64, so a seeded run follows the reference's stream of random numbers.
  * --init-mask must be K x T x F (the reference's layout); another rank, class count or size
    raises ValueError before anything runs.
  * --num-classes is limited to 4 (the kernels' instantiations).
  * an utterance whose eigen-iteration does not converge logs "... Failed" and writes nothing,
    the reference's numpy.linalg.LinAlgError branch.
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
from setk_b200.libs.data_handler import NumpyReader, NumpyWriter, ScriptReader, WaveReader  # noqa: E402
from setk_b200.libs.opts import StftParser, strtobool  # noqa: E402
from setk_b200.libs.utils import default_device, forward_stft, get_logger, get_plan, nextpow2  # noqa: E402

logger = get_logger(__name__)


def train_utterance(samps, args, init_mask, dev):
    """samps C x N float32 -> (masks K x T x F float32 numpy, converged)."""
    C, N = samps.shape
    n_fft = nextpow2(args.frame_len) if args.round_power_of_two else args.frame_len
    K, F = args.num_classes, n_fft // 2 + 1
    tile = n_fft in (512, 1024) and args.frame_hop % 4 == 0 and args.frame_hop <= n_fft
    audio = torch.from_numpy(np.ascontiguousarray(samps)).to(dev)[None]
    if tile:
        plan = get_plan(C, args.frame_len, args.frame_hop, bool(args.center), bool(args.round_power_of_two),
                        args.window, N, dev)
        T = plan.num_frames(N)
    else:
        stft = torch.stack([
            forward_stft(audio[0, c], frame_len=args.frame_len, frame_hop=args.frame_hop,
                         round_power_of_two=bool(args.round_power_of_two), center=bool(args.center),
                         window=args.window, transpose=False) for c in range(C)
        ])                                                                          # C x F x T
        T = stft.shape[-1]
    permu = None
    if args.solve_permu:
        if F not in _plan.PERMU_PLANS:
            raise ValueError(f"Unsupported num_bins: {F}")
        permu = _plan.PERMU_PLANS[F]
    cgmm_init = bool(args.cgmm_init) and K == 2
    init = None
    if init_mask is not None:
        init = np.asarray(init_mask, dtype=np.float64)
        if init.shape != (K, T, F):
            raise ValueError(f"--init-mask must be K x T x F = {(K, T, F)}, got {init.shape}")
        logger.info("Using external mask to initialize cacgmm")
    elif not cgmm_init:
        g = np.random.uniform(size=[K, F, T])                                       # cluster.py:509-512
        init = np.transpose(g / np.sum(g, 0, keepdims=True), (0, 2, 1))
        logger.info(f"Random initialized, num_classes = {K}")
    if init is not None:
        init = torch.from_numpy(np.ascontiguousarray(init))[None].to(dev)
    kw = dict(init_gamma=init, cgmm_init=cgmm_init, update_alpha=bool(args.update_alpha), permu_plan=permu)
    if tile:
        masks, status = plan.cacgmm_masks(audio, K, args.num_iters, **kw)
    else:
        masks, status = _plan.cacgmm_from_stft(stft[None], K, args.num_iters, **kw)
    if permu is not None:
        logger.info("Permutation alignment done on each frequency")
    return masks[0].cpu().numpy(), int(status.abs().sum()) == 0


def run(args):
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
                init_mask = init_mask_reader[key]          # K x T x F
            masks, ok = train_utterance(np.asarray(samps, dtype=np.float32), args, init_mask, dev)
            if not ok:
                logger.warning(f"Training utterance {key} ... Failed")
                continue
            num_done += 1
            writer.write(key, masks.astype(np.float32))
            logger.info(f"Training utterance {key} ... Done")
    logger.info(f"Train {num_done:d} utterances over {len(wave_reader):d}")


if __name__ == "__main__":
    parser = argparse.ArgumentParser(
        description="Speaker masks estimation using Complex Angular "
        "Central Gaussian Mixture Model (CACGMM)",
        formatter_class=argparse.ArgumentDefaultsHelpFormatter,
        parents=[StftParser.parser])
    parser.add_argument("wav_scp", type=str, help="Multi-channel wave scripts in kaldi format")
    parser.add_argument("dst_dir", type=str, help="Where to dump estimated speech masks")
    parser.add_argument("--num-iters", type=int, default=50, help="Number of iterations to train Cacgmm")
    parser.add_argument("--num-classes", type=int, default=2,
                        help="Number of the cluster used in cacgmm model")
    parser.add_argument("--seed", type=int, default=777, help="Random seed for initialization")
    parser.add_argument("--init-mask", type=str, default="", dest="init_mask",
                        help="Mask scripts for cacgmm initialization")
    parser.add_argument("--cgmm-init", type=strtobool, default=False,
                        help="For 2 classes, using the cgmm init way")
    parser.add_argument("--solve-permu", type=strtobool, default=True,
                        help="If true, solving permutation problems")
    parser.add_argument("--update-alpha", type=strtobool, default=True, help="If true, update alpha in M-step")
    parser.add_argument("--mask-format", type=str, dest="fmt", default="numpy", choices=["kaldi", "numpy"],
                        help="Mask storage format")
    args = parser.parse_args()
    run(args)
