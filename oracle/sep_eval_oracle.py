"""
oracle/sep_eval_oracle.py -- the separation metrics in numpy / scipy float64, written from their
definitions (no mir_eval on this machine):

  * bss_eval_sources: BSS-Eval v3 sources criteria (Vincent, Gribonval & Fevotte 2006) the way
    mir_eval.separation.bss_eval_sources computes them -- correlations from zero-padded FFTs, the block
    Toeplitz normal equations G c = D, np.linalg.solve with an lstsq fallback, the FIR projections, the
    energy ratios, and the permutation that maximises the mean SIR (first in itertools order);
  * explicit_projection: the same projections from the dense matrix of delayed references and
    np.linalg.lstsq -- an independent route to the definition, for short signals;
  * si_snr: libs/metric.py's formula in float64.
"""
import itertools

import numpy as np
import scipy.fft
import scipy.linalg
import scipy.signal

FLEN = 512


def _fft_project(refs, est, flen):
    """least-squares projection of est onto the delayed copies of refs (N, S): mir_eval's FFT route"""
    nsrc, nsampl = refs.shape
    refs = np.hstack((refs, np.zeros((nsrc, flen - 1))))
    est = np.hstack((est, np.zeros(flen - 1)))
    n_fft = int(2 ** np.ceil(np.log2(nsampl + flen - 1.0)))
    sf = scipy.fft.fft(refs, n=n_fft, axis=1)
    sef = scipy.fft.fft(est, n=n_fft)
    G = np.zeros((nsrc * flen, nsrc * flen))
    for i in range(nsrc):
        for j in range(nsrc):
            ssf = np.real(scipy.fft.ifft(sf[i] * np.conj(sf[j])))
            ss = scipy.linalg.toeplitz(np.hstack((ssf[0], ssf[-1:-flen:-1])), r=ssf[:flen])
            G[i * flen:(i + 1) * flen, j * flen:(j + 1) * flen] = ss
            G[j * flen:(j + 1) * flen, i * flen:(i + 1) * flen] = ss.T
    D = np.zeros(nsrc * flen)
    for i in range(nsrc):
        ssef = np.real(scipy.fft.ifft(sf[i] * np.conj(sef)))
        D[i * flen:(i + 1) * flen] = np.hstack((ssef[0], ssef[-1:-flen:-1]))
    try:
        C = np.linalg.solve(G, D).reshape(flen, nsrc, order="F")
    except np.linalg.LinAlgError:
        C = np.linalg.lstsq(G, D, rcond=None)[0].reshape(flen, nsrc, order="F")
    sproj = np.zeros(nsampl + flen - 1)
    for i in range(nsrc):
        sproj += scipy.signal.fftconvolve(C[:, i], refs[i])[:nsampl + flen - 1]
    return sproj


def explicit_projection(refs, est, flen):
    """the same projection from A = [delayed copies of every reference] and np.linalg.lstsq"""
    refs = np.atleast_2d(np.asarray(refs, np.float64))
    nsrc, nsampl = refs.shape
    n = nsampl + flen - 1
    A = np.zeros((n, nsrc * flen))
    for i in range(nsrc):
        for a in range(flen):
            A[a:a + nsampl, i * flen + a] = refs[i]
    y = np.zeros(n)
    y[:nsampl] = est
    c = np.linalg.lstsq(A, y, rcond=None)[0]
    return A @ c


def _safe_db(num, den):
    if den == 0:
        return np.inf
    return 10 * np.log10(num / den)


def criteria(refs, ests, flen=FLEN, project=_fft_project):
    """(sdr, sir, sar) as (N, N) float64 arrays, [estimate j, reference i]"""
    refs = np.asarray(refs, np.float64)
    ests = np.asarray(ests, np.float64)
    N, S = refs.shape
    out = np.zeros((3, N, N))
    for j in range(N):
        e = np.hstack((ests[j], np.zeros(flen - 1)))
        p_all = project(refs, ests[j], flen)
        for i in range(N):
            p_spat = project(refs[i:i + 1], ests[j], flen)
            out[0, j, i] = _safe_db(np.sum(p_spat ** 2), np.sum((e - p_spat) ** 2))
            out[1, j, i] = _safe_db(np.sum(p_spat ** 2), np.sum((p_all - p_spat) ** 2))
            out[2, j, i] = _safe_db(np.sum(p_all ** 2), np.sum((e - p_all) ** 2))
    return out


def best_permutation(sir):
    """mir_eval's rule: the permutation maximising mean(sir[perm[k], k]), first in itertools order"""
    N = sir.shape[0]
    perms = list(itertools.permutations(range(N)))
    means = [np.mean(sir[list(p), np.arange(N)]) for p in perms]
    return np.asarray(perms[int(np.argmax(means))])


def bss_eval_sources(reference_sources, estimated_sources, compute_permutation=True, flen=FLEN,
                     project=_fft_project):
    """(sdr, sir, sar, perm) like mir_eval.separation.bss_eval_sources (no input validation)"""
    ref = np.atleast_2d(np.asarray(reference_sources, np.float64))
    est = np.atleast_2d(np.asarray(estimated_sources, np.float64))
    crit = criteria(ref, est, flen, project)
    N = ref.shape[0]
    popt = best_permutation(crit[1]) if compute_permutation else np.arange(N)
    idx = (popt, np.arange(N))
    return crit[0][idx], crit[1][idx], crit[2][idx], popt


def si_snr(x, s, eps=1e-8, remove_dc=True):
    """libs/metric.py si_snr in float64"""
    x = np.asarray(x, np.float64)
    s = np.asarray(s, np.float64)
    if remove_dc:
        x = x - np.mean(x)
        s = s - np.mean(s)
    t = np.inner(x, s) * s / (np.linalg.norm(s, 2) ** 2 + eps)
    n = x - t
    return 20 * np.log10(np.linalg.norm(t, 2) / (np.linalg.norm(n, 2) + eps) + eps)
