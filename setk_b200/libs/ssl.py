"""
setk_b200.libs.ssl -- GPU mirror of the reference's sound source localisation
(scripts/sptk/libs/ssl.py): the same function names, argument names, defaults,
array axes and return types; the arithmetic runs in libsetk_b200.so
(csrc/ssl.cuh: setk_ssl).  No CPU path.

    ml_ssl     ssl.py:12-43    maximum likelihood
    srp_ssl    ssl.py:46-77    SRP-PHAT over microphone pairs
    music_ssl  ssl.py:80-110   MUSIC

Inputs may be numpy arrays or torch tensors: stft M x T x F complex, sv A x M x F
complex (as compute_steer_vector.py writes it), mask T x F (or N x T x F for
ml_ssl).  The index comes back as numpy's argmax / argmin gives it: an integer,
or an array of N indices for a 3-D mask.  return_scores=True also returns the
score vector (A,) or (N, A) the index is taken from, float64, as a numpy array
for numpy input and a tensor otherwise.

Differences from the reference, all deliberate:
  * the mask is taken as float32 (NumpyReader masks are float32 .npy files);
  * srp_ssl uses the correctly rounded float32 phase of every STFT cell, where
    numpy's vectorised float32 arctan2 may be an ulp or two away, and sums
    cos(o - r) as cos o cos r + sin o sin r with the masked frame sum taken
    first (DESIGN.md section 4, K10);
  * music_ssl builds the covariance and its principal eigenvector in float64
    for every mask dtype (the reference runs eigh in complex64 when the mask is
    float32).
"""
import numpy as np
import torch

from .. import plan as _plan
from .utils import default_device

__all__ = ["ml_ssl", "srp_ssl", "music_ssl"]


def _dev(*arrays):
    for a in arrays:
        if torch.is_tensor(a) and a.device.type == "cuda":
            return a.device
    return default_device()


def _run(backend, stft, sv, mask, return_scores, pairs=None, **kwargs):
    was_numpy = not torch.is_tensor(stft)
    dev = _dev(stft, sv, mask)
    S = torch.as_tensor(stft, device=dev)
    if S.dim() != 3:
        raise ValueError(f"stft must be M x T x F, got {tuple(S.shape)}")
    S = S.transpose(1, 2)[None]                                   # 1 x M x F x T
    m = None
    squeeze = True
    if mask is not None:
        m = torch.as_tensor(mask, device=dev)
        if m.dim() == 3:
            squeeze = False
            m = m[None]                                           # 1 x N x T x F
        else:
            m = m[None, None]
    scores, index = _plan.ssl(S, torch.as_tensor(sv, device=dev), backend=backend, mask=m, pairs=pairs,
                              **kwargs)
    idx = index[0, :, 0].cpu().numpy().astype(np.intp)
    sc = scores[0, :, 0]
    if squeeze:
        idx, sc = idx[0], sc[0]
    if not return_scores:
        return idx
    return idx, (sc.cpu().numpy() if was_numpy else sc)


def ml_ssl(stft, sv, compression=0, eps=1e-8, norm=False, mask=None, return_scores=False):
    """
    Maximum likelihood SSL
    Arguments:
        stft: STFT transform result, M x T x F
        sv: steer vector in each directions, A x M x F
        norm: normalze STFT or not
        mask: TF-mask for source, T x F x (N)
    Return:
        index: DoA index
    """
    return _run("ml", stft, sv, mask, return_scores, compression=compression, eps=eps, normalize=norm)


def srp_ssl(stft, sv, srp_pair=None, mask=None, return_scores=False):
    """
    Do SRP-PHAT based SSL
    Arguments:
        stft: STFT transform result, M x T x F
        sv: steer vector in each directions, A x M x F
        srp_pair: index pair to compute srp response
        mask: TF-mask for source, T x F
    Return:
        index: DoA index
    """
    if srp_pair is None:
        raise ValueError("srp_pair cannot be None, (list, list)")
    index_l, index_r = srp_pair
    pairs = list(zip(np.atleast_1d(index_l).tolist(), np.atleast_1d(index_r).tolist()))
    return _run("srp", stft, sv, mask, return_scores, pairs=pairs)


def music_ssl(stft, sv, mask=None, return_scores=False):
    """
    Do MUSIC based SSL
    Arguments:
        stft: STFT transform result, M x T x F
        sv: steer vector in each directions, A x M x F
        mask: TF-mask for source, T x F
    Return:
        index: DoA index
    """
    return _run("music", stft, sv, mask, return_scores)
