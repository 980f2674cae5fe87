"""
Separation metrics on libsetk_b200's kernels: the reference's libs/metric.py (si_snr, permute_si_snr;
permute_ed, which needs editdistance, is not ported) and mir_eval.separation.bss_eval_sources, which
the reference's compute_sdr.py imports.  Every score is computed on the device in fp64
(setk_b200.plan.si_snr / bss_eval); the permutation search runs here over the N x N matrices.

The *_batch forms take lists of utterances of any lengths, run them in device batches of at most
`batch_size` utterances grouped by length, and return one result per utterance in input order.
"""
import itertools

import numpy as np
import torch

from .. import _lib
from .. import plan as _plan
from .utils import default_device

MAX_SOURCES = 100   # mir_eval.separation.MAX_SOURCES (the kernels take at most 8)


def _to_device(arrays, dev):
    """(B, N, S_max) float32 tensor of zero-padded utterances and their lengths"""
    lens = np.array([a.shape[-1] for a in arrays], dtype=np.int32)
    N = arrays[0].shape[0]
    buf = np.zeros((len(arrays), N, int(lens.max())), dtype=np.float32)
    for b, a in enumerate(arrays):
        buf[b, :, :a.shape[-1]] = a
    return torch.from_numpy(buf).to(dev), lens


def first_failure(items, check):
    """(index, exception) of the first item for which check(item) raises, else (len(items), None)"""
    for k, item in enumerate(items):
        try:
            check(item)
        except Exception as err:  # noqa: BLE001 -- re-raised by the caller after the earlier items
            return k, err
    return len(items), None


def _batches(lengths, batch_size):
    """index groups of similar length, each of at most batch_size (every index alone when it is 0)"""
    order = sorted(range(len(lengths)), key=lambda k: (lengths[k], k))
    size = max(1, int(batch_size))
    return [order[k:k + size] for k in range(0, len(order), size)]


def si_snr_matrix_batch(xlists, slists, remove_dc=True, eps=1e-8, batch_size=64):
    """
    For every utterance u, the (N, N) float64 matrix si_snr(xlists[u][j], slists[u][i]) at [j, i].
    xlists, slists: per utterance an (N, S_u) array (or a list of N equal-length vectors).
    """
    xs = [np.atleast_2d(np.asarray(x, dtype=np.float32)) for x in xlists]
    ss = [np.atleast_2d(np.asarray(s, dtype=np.float32)) for s in slists]
    for x, s in zip(xs, ss):
        if x.shape != s.shape:
            raise ValueError(f"si_snr: estimate {x.shape} and reference {s.shape} differ in shape")
    out = [None] * len(xs)
    dev = default_device()
    for group in _batches([x.shape[-1] for x in xs], batch_size):
        est, lens = _to_device([xs[k] for k in group], dev)
        ref, _ = _to_device([ss[k] for k in group], dev)
        m = _plan.si_snr(est, ref, lens, remove_dc=remove_dc, eps=eps).cpu().numpy()
        for r, k in enumerate(group):
            out[k] = m[r]
    return out


def si_snr(x, s, eps=1e-8, remove_dc=True):
    """
    Compute Si-SNR
    Arguments:
        x: vector, enhanced/separated signal
        s: vector, reference signal (ground truth)
    """
    x, s = np.asarray(x), np.asarray(s)
    if x.ndim != 1 or s.ndim != 1 or x.shape != s.shape:
        raise ValueError(f"si_snr needs two vectors of one length, got {x.shape} and {s.shape}")
    return float(si_snr_matrix_batch([x[None]], [s[None]], remove_dc=remove_dc, eps=eps)[0][0, 0])


def best_mean_permutation(score):
    """(best mean of score[k, perm[k]], perm) over itertools.permutations order, first maximum kept"""
    N = score.shape[0]
    best, best_perm = None, None
    for order in itertools.permutations(range(N)):
        avg = sum([score[k, order[k]] for k in range(N)]) / N
        if best is None or avg > best:
            best, best_perm = avg, order
    return best, best_perm


def permute_si_snr(xlist, slist, align=False):
    """
    Compute Si-SNR between N pairs
    Arguments:
        x: list[vector], enhanced/separated signal
        s: list[vector], reference signal (ground truth)
    """
    N = len(xlist)
    if N != len(slist):
        raise RuntimeError("size do not match between xlist " + f"and slist: {N} vs {len(slist)}")
    m = si_snr_matrix_batch([np.stack(xlist)], [np.stack(slist)])[0]
    best, perm = best_mean_permutation(m)
    return (best, perm) if align else best


def validate(reference_sources, estimated_sources):
    """mir_eval.separation.validate's checks and messages (ValueError)"""
    if reference_sources.shape != estimated_sources.shape:
        raise ValueError("The shape of estimated sources and the true sources should match.  "
                         f"reference_sources.shape = {reference_sources.shape}, "
                         f"estimated_sources.shape = {estimated_sources.shape}")
    if reference_sources.ndim > 3 or estimated_sources.ndim > 3:
        raise ValueError("The number of dimensions is too high (must be less than 3). "
                         f"reference_sources.ndim = {reference_sources.ndim}, "
                         f"estimated_sources.ndim = {estimated_sources.ndim}")
    if reference_sources.size and np.any(np.all(reference_sources == 0, axis=-1)):
        raise ValueError(SILENT_REFERENCE)
    if estimated_sources.size and np.any(np.all(estimated_sources == 0, axis=-1)):
        raise ValueError(SILENT_ESTIMATE)
    if estimated_sources.shape[0] > MAX_SOURCES or reference_sources.shape[0] > MAX_SOURCES:
        raise ValueError("The supplied matrices should be of shape (nsrc, nsampl) but "
                         f"reference_sources.shape[0] = {reference_sources.shape[0]} and "
                         f"estimated_sources.shape[0] = {estimated_sources.shape[0]} which is greater than "
                         f"mir_eval.separation.MAX_SOURCES = {MAX_SOURCES}.  To override this check, set "
                         "mir_eval.separation.MAX_SOURCES to a larger value.")


SILENT_REFERENCE = ("All the reference sources should be non-silent (not all-zeros), but at least one of the "
                    "reference sources is all 0s, which introduces ambiguity to the evaluation. (Otherwise we "
                    "can add infinitely many all-zero sources.)")
SILENT_ESTIMATE = ("All the estimated sources should be non-silent (not all-zeros), but at least one of the "
                   "estimated sources is all 0s. Since we require each reference source to be non-silent, "
                   "having a silent estimated source will result in an underdetermined system.")


def bss_eval_matrix_batch(references, estimates, flen=512, batch_size=64):
    """
    For every utterance u (references[u], estimates[u]: (N, S_u) arrays, validated like mir_eval), the
    (3, N, N) float64 SDR / SIR / SAR of estimate j against reference i at [:, j, i].
    """
    refs = [np.atleast_2d(np.asarray(r)) for r in references]
    ests = [np.atleast_2d(np.asarray(e)) for e in estimates]
    for r, e in zip(refs, ests):
        validate(r, e)
    out = [None] * len(refs)
    dev = default_device()
    for group in _batches([r.shape[-1] for r in refs], batch_size):
        ref, lens = _to_device([refs[k].astype(np.float32) for k in group], dev)
        est, _ = _to_device([ests[k].astype(np.float32) for k in group], dev)
        crit, _, status = _plan.bss_eval(est, ref, lens, flen=flen)
        crit, status = crit.cpu().numpy(), status.cpu().numpy()
        for r, k in enumerate(group):
            if status[r] & _lib.ST_SILENT:   # float32 rounding made a source all zeros
                raise ValueError(SILENT_REFERENCE if np.any(np.all(ref[r].cpu().numpy() == 0, axis=-1))
                                 else SILENT_ESTIMATE)
            out[k] = crit[r]
    return out


def _select(crit, compute_permutation):
    N = crit.shape[-1]
    dum = np.arange(N)
    if compute_permutation:
        perms = list(itertools.permutations(range(N)))
        mean_sir = np.array([np.mean(crit[1][list(p), dum]) for p in perms])
        popt = np.asarray(perms[int(np.argmax(mean_sir))])
    else:
        popt = dum
    idx = (popt, dum)
    return crit[0][idx], crit[1][idx], crit[2][idx], popt


def bss_eval_sources_batch(references, estimates, compute_permutation=True, batch_size=64):
    """bss_eval_sources of every (references[u], estimates[u]), in input order"""
    return [_select(c, compute_permutation) for c in bss_eval_matrix_batch(references, estimates,
                                                                              batch_size=batch_size)]


def bss_eval_sources(reference_sources, estimated_sources, compute_permutation=True):
    """
    mir_eval.separation.bss_eval_sources: (sdr, sir, sar, perm) for reference_sources and
    estimated_sources of shape (nsrc, nsampl) (or (nsampl,)), with mir_eval's ValueErrors; with
    compute_permutation the estimates are matched to the references by the best mean SIR, and perm[k]
    is the estimate matched to reference k.
    """
    ref = np.asarray(reference_sources)
    est = np.asarray(estimated_sources)
    if est.ndim == 1:
        est = est[np.newaxis, :]
    if ref.ndim == 1:
        ref = ref[np.newaxis, :]
    validate(ref, est)
    if ref.size == 0 or est.size == 0:
        return np.array([]), np.array([]), np.array([]), np.array([])
    return bss_eval_sources_batch([ref], [est], compute_permutation)[0]
