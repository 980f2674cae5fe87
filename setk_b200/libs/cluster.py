"""
setk_b200.libs.cluster -- GPU mirror of the reference's CGMM and CACGMM trainers
(scripts/sptk/libs/cluster.py:396-465 and 468-535, with the model classes 94-393 behind them).

    trainer = CgmmTrainer(obs, num_classes, gamma=None, cgmm=None, update_alpha=False)
    trainer = CacgmmTrainer(obs, num_classes, gamma=None, cacgmm=None, cgmm_init=False, update_alpha=True)
    gamma = trainer.train(num_iters)          # K x F x T posteriors

Same constructor / method names, argument meaning and array axes as the
reference; the arithmetic runs in libsetk_b200.so (setk_cgmm_stft: bin-major EM in
fp64, csrc/cgmm.cu).  There is no CPU path: without the CUDA library the import
of the loader fails.

Differences from the reference, all deliberate:
  * obs may be a torch tensor (any device; moved to the default CUDA device) or a
    numpy array; `train` returns the same kind.  Posteriors come back as float32
    (the reference computes float64 and its CLI stores float32).
  * the K = 2 start accumulates sum_t y y^H / T in fp64; the reference's einsum is
    complex64 there (cluster.py:419-420).  See oracle/cgmm_oracle.py for what that
    does to the masks.
  * more than two classes need `gamma` (the reference draws np.random.uniform; draw
    it with numpy and pass it in to reproduce a seeded run exactly).
  * `cgmm=<pickle path>` (resume) raises: the reference opens the pickle in text
    mode, which cannot work under Python 3 (cluster.py:455-457).
  * the per-iteration log value Q is not computed.
  * CacgmmTrainer runs setk_cacgmm_stft (csrc/cgmm.cu with ACG = true) and draws its random
    start with np.random.uniform in the constructor, as the reference does, so np.random.seed
    reproduces a reference run.  Its start is float64 and its masks come back float32;
    `cacgmm=<pickle path>` raises like `cgmm=`; a non-converged eigen-iteration raises
    numpy.linalg.LinAlgError, as the reference's eigh would.
  * permu_aligner below is host numpy; plan.permu_align is its device form.
"""
import numpy as np
import torch

from .. import plan as _plan
from .utils import EPSILON, default_device, get_logger

logger = get_logger(__name__)

__all__ = ["CgmmTrainer", "CacgmmTrainer", "permu_aligner", "norm_observation", "supported_plan"]

# frequency sub-band schedule of the permutation aligner: (iterations, first bin, end bin)
supported_plan = _plan.PERMU_PLANS


def norm_observation(mat, axis=-1, eps=EPSILON):
    """Unit 2-norm along `axis`, the norm floored at eps (cluster.py:39-45)."""
    mat = np.asarray(mat)
    return mat / np.maximum(np.linalg.norm(mat, axis=axis, keepdims=True), eps)


def _best_permutation(score):
    """argmax over permutations of sum_k score[k, perm[k]] (K <= 4: enumerate)."""
    from itertools import permutations
    K = score.shape[0]
    best, best_val = None, -np.inf
    for perm in permutations(range(K)):
        val = sum(score[k, perm[k]] for k in range(K))
        if val > best_val + 1e-15:
            best, best_val = perm, val
    return np.asarray(best)


def permu_aligner(masks, transpose=False):
    """
    Frequency permutation alignment of K x T x F masks (cluster.py:48-91): correlate
    every bin's normalised mask tracks with the centroid of a sub-band and re-order
    the classes of the bin to the best assignment, sub-band by sub-band.
    Host-side (numpy): K x K assignments over F bins, outside the GPU hot path.
    """
    masks = np.asarray(masks)
    if masks.ndim != 3:
        raise RuntimeError("Expect 3D TF-masks, K x T x F or K x F x T")
    if transpose:
        masks = np.transpose(masks, (0, 2, 1))
    K, _, F = masks.shape
    if F not in supported_plan:
        raise ValueError(f"Unsupported num_bins: {F}")
    feature = norm_observation(masks, axis=1)
    order = np.tile(np.arange(K)[:, None], (1, F))          # order[k, f]: source class of slot k
    for iters, lo, hi in supported_plan[F]:
        for _ in range(iters):
            centroid = norm_observation(np.mean(feature[..., lo:hi], axis=-1), axis=-1)   # K x T
            moved = False
            for f in range(lo, hi):
                score = centroid @ norm_observation(feature[..., f], axis=-1).T             # K x K
                perm = _best_permutation(score)
                if np.any(perm != np.arange(K)):
                    feature[..., f] = feature[perm, :, f]
                    order[:, f] = order[perm, f]
                    moved = True
            if not moved:
                break
    out = np.empty_like(masks)
    for f in range(F):
        out[..., f] = masks[order[:, f], :, f]
    return out


def _complex_obs(obs, who):
    """obs M x F x T (or B x M x F x T) -> (complex64 B x M x F x T on a CUDA device, was numpy, batched)"""
    numpy = isinstance(obs, np.ndarray)
    obs = torch.as_tensor(obs)
    if not torch.is_complex(obs):
        raise RuntimeError(f"{who} expects a complex STFT, M x F x T")
    batched = obs.dim() == 4
    if obs.dim() == 3:
        obs = obs[None]
    if obs.dim() != 4:
        raise RuntimeError(f"Expect M x F x T observations, got {tuple(obs.shape)}")
    dev = obs.device if obs.device.type == "cuda" else default_device()
    return obs.to(dev).to(torch.complex64).contiguous(), numpy, batched


class CgmmTrainer(object):
    """
    CGMM trainer (cluster.py:396-465).
        obs    mixture STFT, M x F x T complex (or B x M x F x T for a batch)
        gamma  starting posteriors: None (2 classes, deterministic start), F x T
               (2 classes: stacked with its complement) or K x F x T
    """

    def __init__(self, obs, num_classes, gamma=None, cgmm=None, update_alpha=False):
        if cgmm is not None:
            raise NotImplementedError("resuming from a pickled Cgmm is not supported "
                                      "(broken in the reference: text-mode pickle, cluster.py:455)")
        self.obs, self._numpy, self._batched = _complex_obs(obs, "CgmmTrainer")
        dev = self.obs.device
        B, M, F, T = self.obs.shape
        self.num_classes = int(num_classes)
        self.update_alpha = bool(update_alpha)
        logger.info(f"CGMM instance: F = {F:d}, T = {T:}, M = {M}")
        self._init = None
        if gamma is not None:
            g = torch.as_tensor(gamma).to(dev).to(torch.float32)
            if self.num_classes == 2 and g.dim() == (3 if self._batched else 2):
                g = torch.stack([g, 1 - g], dim=-3)                  # cluster.py:428-429
            if not self._batched:
                g = g[None]
            if tuple(g.shape) != (B, self.num_classes, F, T):
                raise RuntimeError(f"gamma must be K x F x T = {(self.num_classes, F, T)}, "
                                   f"got {tuple(g.shape[1:])}")
            self._init = g.transpose(-1, -2).contiguous()            # library layout K x T x F
        elif self.num_classes != 2:
            raise RuntimeError("more than 2 classes need starting posteriors `gamma` "
                               "(draw them with numpy to reproduce a seeded reference run)")
        self._iters = 0
        self.gamma = None

    def train(self, num_iters):
        """
        EM iterations; returns the posteriors K x F x T.  Calling it again continues:
        the run is deterministic, so it is redone with the accumulated count.
        """
        self._iters += int(num_iters)
        masks, status = _plan.cgmm_from_stft(self.obs, self.num_classes, self._iters,
                                             init_gamma=self._init, update_alpha=self.update_alpha)
        bad = status.nonzero().flatten().tolist()
        if bad:
            raise RuntimeError(f"CGMM: eigen-iteration did not converge for batch entries {bad}")
        gamma = masks.transpose(-1, -2)                              # K x F x T like the reference
        if not self._batched:
            gamma = gamma[0]
        self.gamma = gamma.cpu().numpy() if self._numpy else gamma
        return self.gamma


class CacgmmTrainer(object):
    """
    CACGMM trainer (cluster.py:468-535).
        obs        mixture STFT, M x F x T complex (or B x M x F x T for a batch)
        gamma      starting posteriors K x F x T (B x K x F x T), used as given; None draws
                   np.random.uniform(size=[K, F, T]) here (per utterance, in batch order) and
                   normalises it over classes, unless cgmm_init with 2 classes
        cgmm_init  with 2 classes: the start B_0 = sum_t z z^H / T, B_1 = I and one E-step
    """

    def __init__(self, obs, num_classes, gamma=None, cacgmm=None, cgmm_init=False, update_alpha=True):
        if cacgmm is not None:
            raise NotImplementedError("resuming from a pickled Cacgmm is not supported "
                                      "(broken in the reference: text-mode pickle, cluster.py:520-522)")
        self.obs, self._numpy, self._batched = _complex_obs(obs, "CacgmmTrainer")
        B, M, F, T = self.obs.shape
        self.num_classes = K = int(num_classes)
        self.update_alpha = bool(update_alpha)
        self.cgmm_init = bool(cgmm_init) and K == 2
        logger.info(f"CACGMM instance: F = {F:d}, T = {T:}, M = {M}")
        self._init = None
        if gamma is not None:
            g = torch.as_tensor(gamma).to(self.obs.device).to(torch.float64)
            if not self._batched:
                g = g[None]
            if tuple(g.shape) != (B, K, F, T):
                raise RuntimeError(f"gamma must be K x F x T = {(K, F, T)}, got {tuple(g.shape[1:])}")
            self._init = g.transpose(-1, -2).contiguous()            # library layout K x T x F
        elif self.cgmm_init:
            logger.info("Using cgmm init for num_classes = 2")
        else:
            draws = []
            for _ in range(B):                                        # cluster.py:509-512
                g = np.random.uniform(size=[K, F, T])
                draws.append(np.transpose(g / np.sum(g, 0, keepdims=True), (0, 2, 1)))
            self._init = torch.from_numpy(np.ascontiguousarray(np.stack(draws))).to(self.obs.device)
            logger.info(f"Random initialized, num_classes = {K}")
        self._iters = 0
        self.gamma = None

    def train(self, num_iters):
        """
        EM iterations; returns the posteriors K x F x T.  Calling it again continues: the run is
        deterministic, so it is redone with the accumulated count.
        """
        self._iters += int(num_iters)
        masks, status = _plan.cacgmm_from_stft(self.obs, self.num_classes, self._iters, init_gamma=self._init,
                                               cgmm_init=self.cgmm_init, update_alpha=self.update_alpha)
        bad = status.nonzero().flatten().tolist()
        if bad:
            raise np.linalg.LinAlgError(f"CACGMM: eigen-iteration did not converge for batch entries {bad}")
        gamma = masks.transpose(-1, -2)                              # K x F x T like the reference
        if not self._batched:
            gamma = gamma[0]
        self.gamma = gamma.cpu().numpy() if self._numpy else gamma
        return self.gamma
