"""
oracle/cacgmm_oracle.py -- CPU restatement of the reference's CACGMM mask estimator and of its
frequency permutation aligner.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Not imported by the product.

What it restates (scripts/sptk/libs/cluster.py)
  * 39-45    norm_observation: z = y / max(|y|_2, eps) over channels
  * 94-136   Covariance, in the precision of the matrix it is given
  * 290-337  CacgDistribution.update_parameters / log_pdf
               B_k   = M sum_t (gamma_k / kappa_k) z z^H / max(sum_t gamma_k, eps)
               kappa = max(|z^H B_k^-1 z|, eps)
               log A = -M log kappa - log det B_k
  * 340-393  Cacgmm.update / predict (kernel = kappa of the last E-step, ones at a given start)
  * 468-535  CacgmmTrainer: the random (np.random.uniform) or given start, no E-step before the
             first M-step; or, with cgmm_init and 2 classes, B_0 = sum_t z z^H / T, B_1 = I and
             one E-step
  * 48-91    permu_aligner, with every decision's margin (best minus second-best score)
  * estimate_cacgmm_masks.py:40-63  K x F x T -> K x T x F

Arithmetic follows numpy's type promotion from two choices:
  obs_dtype    complex64 reproduces the reference, whose norm_observation of a complex64 STFT is
               complex64; complex128 (the default) normalises in fp64, as the kernels do
  start_dtype  complex64 reproduces the reference's cgmm_init start, where np.eye(dtype=obs.dtype)
               keeps the first factor and E-step in single precision; complex128 is the default
With both complex64 it reproduces the reference's masks to float32 storage rounding
(tests/golden/PINNING_cacgmm.json).
"""
import numpy as np

from oracle.cgmm_oracle import EPSILON

PERMU_PLANS = {
    257: [(20, 70, 170), (2, 90, 190), (2, 50, 150), (2, 110, 210), (2, 30, 130), (2, 130, 230),
          (2, 0, 110), (2, 150, 257)],
    513: [(20, 100, 200), (2, 120, 220), (2, 80, 180), (2, 140, 240), (2, 60, 160), (2, 160, 260),
          (2, 40, 140), (2, 180, 280), (2, 0, 120)] +
         [(2, lo, lo + 100) for lo in range(200, 400, 20)] + [(2, 400, 513)],
}


def norm_observation(mat, axis=-1, eps=EPSILON):
    """cluster.py:39-45 (the dtype of `mat` is kept, as numpy keeps it)."""
    return mat / np.maximum(np.linalg.norm(mat, axis=axis, keepdims=True), eps)


def _factor(covar):
    """Covariance(covar) of cluster.py:99-113 in covar's own precision: (B^-1, log det K x F x 1)."""
    c = (covar + np.einsum("...xy->...yx", covar.conj())) / 2
    w, v = np.linalg.eigh(c)
    w = w / np.maximum(np.amax(w, axis=-1, keepdims=True), EPSILON)
    w = np.maximum(w, EPSILON)
    return np.einsum("...xy,...y,...zy->...xz", v, 1 / w, v.conj()), np.sum(np.log(w), axis=-1, keepdims=True)


def _predict(z, B_inv, log_det, alpha):
    """Cacgmm.predict without Q (cluster.py:367-393): (gamma, kernel)."""
    M = z.shape[1]
    kernel = np.einsum("...xt,...xy,...yt->...t", z.conj(), B_inv, z)
    kernel = np.maximum(np.abs(kernel), EPSILON)
    log_pdf = -M * np.log(kernel) - log_det
    log_pdf = log_pdf - np.amax(log_pdf, 0, keepdims=True)
    nominator = np.exp(log_pdf) * alpha[..., None]
    return nominator / np.maximum(np.sum(nominator, 0, keepdims=True), EPSILON), kernel


def cacgmm_posteriors(stft, num_classes=2, num_iters=50, gamma=None, cgmm_init=False, update_alpha=True,
                      obs_dtype=np.complex128, start_dtype=np.complex128):
    """
    CacgmmTrainer(stft, num_classes, gamma, cgmm_init=..., update_alpha=...).train(num_iters).
    stft M x F x T complex; gamma K x F x T (the start, used as given, in its own dtype) or None with
    cgmm_init and 2 classes.  Returns the K x F x T float64 posteriors.
    """
    z = np.einsum("mft->fmt", norm_observation(np.asarray(stft).astype(obs_dtype), axis=0))
    F, M, T = z.shape
    K = num_classes
    alpha = np.ones([K, F]) / K
    if cgmm_init and K == 2:
        zs = z.astype(start_dtype)
        covar = np.stack([np.einsum("...xt,...yt->...xy", zs, zs.conj()) / T,
                          np.stack([np.eye(M, M, dtype=start_dtype) for _ in range(F)])])
        gamma, kernel = _predict(z, *_factor(covar), alpha)
    else:
        if gamma is None:
            raise ValueError("a start is needed unless cgmm_init with 2 classes")
        gamma = np.asarray(gamma)     # its dtype kept: a float32 mask makes the first sums float32, as there
        kernel = np.ones([K, F, T])
    for _ in range(num_iters):
        den = np.sum(gamma, -1, keepdims=True)
        covar = M * np.einsum("...t,...xt,...yt->...xy", gamma / kernel, z, z.conj())
        covar = covar / np.maximum(den[..., None], EPSILON)
        B_inv, log_det = _factor(covar)
        if update_alpha:
            alpha = np.mean(gamma, -1)
        gamma, kernel = _predict(z, B_inv, log_det, alpha)
    return gamma


def permu_align(masks, plan=None):
    """
    permu_aligner(masks) (cluster.py:48-91) in float64 on K x T x F masks, with the tie rule of
    setk_b200.libs.cluster._best_permutation.  Returns (aligned K x T x F, mapping K x F,
    margins: best minus second-best permutation score of every bin decision taken, except exact
    ties of all K! scores, such as a silent bin, which keep the order on every implementation).
    """
    from itertools import permutations
    masks = np.asarray(masks, dtype=np.float64)
    K, _, F = masks.shape
    plan = PERMU_PLANS[F] if plan is None else plan
    perms = list(permutations(range(K)))
    feature = norm_observation(masks, axis=1)
    order = np.tile(np.arange(K)[:, None], (1, F))
    margins = []
    for iters, lo, hi in plan:
        for _ in range(iters):
            centroid = norm_observation(np.mean(feature[..., lo:hi], axis=-1), axis=-1)
            moved = False
            for f in range(lo, hi):
                score = centroid @ norm_observation(feature[..., f], axis=-1).T
                vals = [sum(score[k, p[k]] for k in range(K)) for p in perms]
                best, best_val = 0, -np.inf
                for i, v in enumerate(vals):
                    if v > best_val + 1e-15:
                        best, best_val = i, v
                if min(vals) != max(vals):
                    margins.append(best_val - max(v for i, v in enumerate(vals) if i != best))
                perm = np.asarray(perms[best])
                if best != 0:
                    feature[..., f] = feature[perm, :, f]
                    order[:, f] = order[perm, f]
                    moved = True
            if not moved:
                break
    out = np.empty_like(masks)
    for f in range(F):
        out[..., f] = masks[order[:, f], :, f]
    return out, order, np.asarray(margins)
