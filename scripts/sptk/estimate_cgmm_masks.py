#!/usr/bin/env python
# coding=utf-8
"""
Speech & noise mask estimation with a CGMM

Drop-in for the reference's scripts/sptk/estimate_cgmm_masks.py (same positional
arguments, flags, defaults and outputs: <dst_dir>/<key>.npy, float32, T x F for two
classes, K x T x F otherwise; utterances whose .npy exists are skipped), with the
STFT and the EM iterations on libsetk_b200's CUDA kernels (setk_cgmm_masks: tile
STFT into a bin-major workspace, then fp64 covariance / eigen / posterior kernels;
csrc/cgmm.cu).  Frame sizes other than 512 / 1024 points go through the generic
STFT and setk_cgmm_stft.

Notes against the reference:
  * --num-classes > 2 without --init-mask: the reference starts from
    np.random.uniform posteriors after np.random.seed(--seed); the same numbers
    are drawn here with numpy (once per utterance, in file order) and handed to the
    GPU, so a seeded run follows the reference's stream of random numbers.
  * --num-classes is limited to 4 (the kernels' instantiations).
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

from setk_b200 import cgmm_cli  # noqa: E402
from setk_b200.libs.cluster import CgmmTrainer, permu_aligner  # noqa: E402
from setk_b200.libs.opts import StftParser, strtobool  # noqa: E402
from setk_b200.libs.utils import get_logger  # noqa: E402

logger = get_logger(__name__)


def train_utterance(samps, args, init_mask, dev):
    """samps C x N float32 -> the masks to write: K x T x F float32 numpy, T x F for two classes."""
    K = args.num_classes
    try:
        if init_mask is not None:
            logger.info("Using external TF-mask to initialize cgmm")
        audio, plan, stft, T, F = cgmm_cli.observe(samps, args, dev)
        init = None                                                                # K x T x F
        if init_mask is not None:
            init = torch.from_numpy(np.asarray(init_mask, dtype=np.float32)).to(dev)   # T x F or K x T x F
            if init.dim() == 2:
                init = torch.stack([init, 1 - init])                               # cluster.py:428-429
        elif K != 2:
            g = np.random.uniform(size=[K, F, T])                                  # cluster.py:432-434
            g = g / np.sum(g, 0, keepdims=True)
            init = torch.from_numpy(np.transpose(g, (0, 2, 1)).astype(np.float32)).to(dev)
        if plan is not None:
            masks, status = plan.cgmm_masks(audio, K, args.num_iters,
                                            init_gamma=None if init is None else init[None].contiguous(),
                                            update_alpha=bool(args.update_alpha))
            if int(status.abs().sum()) != 0:
                raise RuntimeError("eigen-iteration did not converge")
            masks = masks[0].cpu().numpy()
        else:
            trainer = CgmmTrainer(stft, K, gamma=None if init is None else init.transpose(-1, -2),
                                  update_alpha=bool(args.update_alpha))
            masks = trainer.train(args.num_iters).transpose(-1, -2).cpu().numpy()
        if args.solve_permu:
            masks = permu_aligner(masks)
            logger.info("Permutation alignment done on each frequency")
    except RuntimeError as err:
        raise cgmm_cli.Failed(err) from err
    return masks[0] if K == 2 else masks


if __name__ == "__main__":
    parser = argparse.ArgumentParser(
        description="Speech & Noise mask estimation using CGMM model "
        "(also see: estimate_cacgmm_masks.py)",
        formatter_class=argparse.ArgumentDefaultsHelpFormatter,
        parents=[StftParser.parser])
    parser.add_argument("wav_scp", type=str, help="Multi-channel wave scripts in kaldi format")
    parser.add_argument("dst_dir", type=str, help="Location to dump estimated speech masks")
    parser.add_argument("--num-iters", type=int, default=20,
                        help="Number of iterations to train CGMM parameters")
    parser.add_argument("--num-classes", type=int, default=2,
                        help="Number of the cluster used in cacgmm model")
    parser.add_argument("--seed", type=int, default=777, help="Random seed for initialization")
    parser.add_argument("--init-mask", type=str, default="", dest="init_mask",
                        help="Initial TF-mask for cgmm initialization")
    parser.add_argument("--solve-permu", type=strtobool, default=False,
                        help="If true, solving permutation problems")
    parser.add_argument("--update-alpha", type=strtobool, default=False,
                        help="If true, update alpha in M-step")
    parser.add_argument("--mask-format", type=str, dest="fmt", default="numpy",
                        choices=["kaldi", "numpy"], help="Mask storage format")
    args = parser.parse_args()
    cgmm_cli.run(args, train_utterance)
