"""
setk_b200.libs.beamformer -- drop-in for the mask-based adaptive beamformer part
of the reference's scripts/sptk/libs/beamformer.py on libsetk_b200 kernels.

Same names, argument names, defaults and array axis orders as the reference
(for N: num_mics, F: num_bins, T: num_frames):
    obs (N,F,T), tf_mask (T,F), covariance (F,N,N), weight (F,N), enhanced (F,T)

  do_ban 14-28, solve_pevd 31-63, rank1_constraint 66-84, compute_covar 87-103,
  Beamformer.beamform 220-234, SupervisedBeamformer 237-283,
  OnlineSupervisedBeamformer 286-320, MvdrBeamformer 515-539,
  MpdrBeamformer 542-590, PmwfBeamformer 593-659, GevdBeamformer 662-682,
  OnlineGevdBeamformer 685-703, OnlineMvdrBeamformer 706-728;
  geometry-based (SURVEY.md 8f rank 3): beam_pattern 106-130, diffuse_covar 133-152,
  plane/linear/circular_steer_vector 155-212, FixedBeamformer 323-340, DSBeamformer
  343-377, Linear/CircularDSBeamformer 380-428, Linear/CircularSDBeamformer 431-512.
  Their weights depend on the array geometry only (a few hundred constants per
  direction, computed once on the host like the STFT window); the data path --
  Beamformer.beamform on the observations -- is setk_apply.

numpy in -> numpy out, torch in -> torch out (same device).  Every function
accepts an optional leading batch dimension on its array arguments.

Differences from the reference, all deliberate (SURVEY.md section 0, App. B):
  * eigenvectors follow this library's convention (unit norm, component 0 real
    and >= 0; GEV normalised to w^H Rn w = 1) -- the reference's are defined
    up to a LAPACK-chosen sign per bin;
  * the C x C solves run in float64 whatever the input dtype; results are
    returned as complex64 for complex64/float32 inputs, complex128 otherwise;
  * singular / non-positive-definite covariances raise
    numpy.linalg.LinAlgError (the reference's GEV silently falls back to a
    non-Hermitian eig, beamformer.py:55-58);
  * OnlineSupervisedBeamformer.run takes `ban=` (the reference CLI passes
    `normalize=`, a TypeError, apply_adaptive_beamformer.py:45) and the reset
    flag is cleared after the first chunk (the reference never clears it);
  * MpdrBeamformer.run(ban=True) without whiten computes Rn instead of raising
    UnboundLocalError (beamformer.py:590).
"""
import numpy as np
import torch

from .. import _lib
from .. import plan as _plan
from ..engine import status_message
from .utils import EPSILON, _back, _to_tensor, cmat_abs  # noqa: F401

__all__ = [
    "do_ban", "solve_pevd", "rank1_constraint", "compute_covar", "Beamformer",
    "SupervisedBeamformer", "OnlineSupervisedBeamformer", "MvdrBeamformer", "MpdrBeamformer",
    "PmwfBeamformer", "GevdBeamformer", "OnlineGevdBeamformer", "OnlineMvdrBeamformer",
    "beam_pattern", "diffuse_covar", "plane_steer_vector", "linear_steer_vector",
    "circular_steer_vector", "FixedBeamformer", "DSBeamformer", "LinearDSBeamformer",
    "CircularDSBeamformer", "LinearSDBeamformer", "CircularSDBeamformer"
]


def _complex(x):
    t, was_np = _to_tensor(x)
    if not t.is_complex():
        t = t.to(torch.complex64)
    return t, was_np


def _batched(t, ndim):
    """Add a leading batch axis if `t` has exactly `ndim` dims."""
    if t.dim() == ndim:
        return t.unsqueeze(0), True
    if t.dim() == ndim + 1:
        return t, False
    raise ValueError(f"expected {ndim} or {ndim + 1} dimensions, got {tuple(t.shape)}")


def _check_status(status):
    st = status.cpu().numpy() & _lib.ST_ERROR_MASK        # SETK_ST_REGULARIZED is a warning
    bad = np.nonzero(st)[0]
    if bad.size:
        i = int(bad[0])
        if int(st[i]) & _lib.ST_BAD_REF:
            raise RuntimeError("Reference channel ID exceeds total channels")
        raise np.linalg.LinAlgError(status_message(int(st[i])))


def _solve_dtype(*mats):
    """float64 solve always; complex128 out only if an input is complex128."""
    return torch.complex128 if any(m is not None and m.dtype == torch.complex128
                                   for m in mats) else torch.complex64


def _weights(kind, Rs, Rn=None, Ry=None, **kw):
    Rs, was_np = _complex(Rs)
    Rs, squeeze = _batched(Rs, 3)
    mats = [Rs] + [None if m is None else _batched(_complex(m)[0], 3)[0] for m in (Rn, Ry)]
    dt = _solve_dtype(*mats)
    mats = [None if m is None else m.to(dt) for m in mats]
    w, status, ref = _plan.weights(kind, mats[0], mats[1], mats[2], out_dtype=dt, **kw)
    _check_status(status)
    return _back(w[0] if squeeze else w, was_np)


def do_ban(weight, Rn):
    """
    Do Blind Analytical Normalization(BAN)  (beamformer.py:14-28)
    Arguments: weight F x N, Rn F x N x N.  Return: ban_weight F x N
    """
    w, was_np = _complex(weight)
    w, squeeze = _batched(w, 2)
    R, _ = _complex(Rn)
    R = _batched(R, 3)[0]
    dt = _solve_dtype(w, R)
    out = _plan.ban(w.to(dt), R.to(dt))
    return _back(out[0] if squeeze else out, was_np)


def solve_pevd(Rs, Rn=None):
    """
    Return principle eigenvector of covariance matrix (pair)  (beamformer.py:31-63)
    Arguments: Rs F x N x N, Rn same or None.  Return: pvector F x N
    """
    return _weights(_lib.BF_PEVD, Rs, Rn)


def rank1_constraint(Rs, Rn=None):
    """
    Return generalized rank1 approximation of covariance matrix  (beamformer.py:66-84)
    """
    R, was_np = _complex(Rs)
    R, squeeze = _batched(R, 3)
    Rn_t = None
    if Rn is not None:
        Rn_t, _ = _complex(Rn)
        Rn_t = _batched(Rn_t, 3)[0]
    dt = _solve_dtype(R, Rn_t)
    out, status = _plan.rank1(R.to(dt), None if Rn_t is None else Rn_t.to(dt))
    _check_status(status)
    return _back(out[0] if squeeze else out, was_np)


def compute_covar(obs, tf_mask):
    """
    (beamformer.py:87-103)
    Arguments: tf_mask T x F, obs N x F x T.  Return: covar_mat F x N x N
    """
    x, was_np = _complex(obs)
    x, squeeze = _batched(x, 3)
    m, _ = _to_tensor(tf_mask, torch.float32)
    m = _batched(m, 2)[0]
    R = _plan.covariance(x, m)
    return _back(R[0] if squeeze else R, was_np)


class Beamformer(object):

    def __init__(self):
        pass

    def beamform(self, weight, obs):
        """
        (beamformer.py:220-234)
        Arguments: weight F x N, obs N x F x T.  Return: stft_enhan F x T
        """
        x, was_np = _complex(obs)
        w, _ = _complex(weight)
        x, squeeze = _batched(x, 3)
        w = _batched(w, 2)[0]
        if w.shape[-2] != x.shape[-2] or w.shape[-1] != x.shape[-3]:
            raise ValueError("Input obs do not match with weight, " +
                             f"{tuple(w.shape[-2:])} vs {tuple(x.shape[-3:])}")
        enh = _plan.apply_weights(x, w)
        return _back(enh[0] if squeeze else enh, was_np)


class SupervisedBeamformer(Beamformer):
    """
    BaseClass for TF-mask based beamformer  (beamformer.py:237-283)
    """

    def __init__(self, num_bins):
        super(SupervisedBeamformer, self).__init__()
        self.num_bins = num_bins

    def compute_covar_mat(self, target_mask, obs):
        """
        Arguments: target_mask T x F, obs N x F x T.  Return: covar_mat F x N x N
        """
        if target_mask.shape[-1] != self.num_bins or target_mask.ndim not in (2, 3):
            raise ValueError("Input mask matrix should be shape as " +
                             f"[num_frames x num_bins], now is {tuple(target_mask.shape)}")
        if obs.shape[-2] != target_mask.shape[-1] or obs.shape[-1] != target_mask.shape[-2]:
            raise ValueError("Shape of input obs do not match with " +
                             f"mask matrix, {tuple(obs.shape)} vs {tuple(target_mask.shape)}")
        return compute_covar(obs, target_mask)

    def weight(self, Rs, Rn):
        """
        Need reimplement for different beamformer
        """
        raise NotImplementedError

    def run(self, mask_s, obs, mask_n=None, ban=False):
        """
        Run beamformer based on TF-mask  (beamformer.py:270-283)
        Arguments: mask_s T x F, obs N x F x T.  Returns: stft_enhan F x T
        """
        Rn = self.compute_covar_mat(1 - mask_s if mask_n is None else mask_n, obs)
        Rs = self.compute_covar_mat(mask_s, obs)
        weight = self.weight(Rs, Rn)
        return self.beamform(do_ban(weight, Rn) if ban else weight, obs)


class OnlineSupervisedBeamformer(SupervisedBeamformer):
    """
    Online version of SupervisedBeamformer  (beamformer.py:286-320)
    """

    def __init__(self, num_bins, num_channels, alpha=0.8, normalized_update=False):
        super(OnlineSupervisedBeamformer, self).__init__(num_bins)
        self.covar_mat_shape = (num_bins, num_channels, num_channels)
        self.normalized_update = bool(normalized_update)
        self.reset_stats(alpha=alpha)

    def reset_stats(self, alpha=0.8):
        self.Rs = None
        self.Rn = None
        self.alpha = alpha
        self.reset = True

    def run(self, mask_s, obs, mask_n=None, ban=False):
        Rn = self.compute_covar_mat(1 - mask_s if mask_n is None else mask_n, obs)
        Rs = self.compute_covar_mat(mask_s, obs)
        if tuple(Rs.shape[-3:]) != self.covar_mat_shape:
            raise ValueError(f"covariance shape {tuple(Rs.shape)} vs {self.covar_mat_shape}")
        # update stats.  The reference never clears `reset` (beamformer.py:314-316), so its
        # recursion is R <- alpha R + R_chunk for every chunk; that is the default here.
        # normalized_update=True is the evidently intended R <- alpha R + (1 - alpha) R_chunk
        # after the first chunk (the weights differ only by a per-bin scale of R for MVDR / GEV
        # once the sum has converged, but not during the first chunks).
        phi = 1 if (self.reset or not self.normalized_update) else (1 - self.alpha)
        self.Rs = phi * Rs if self.Rs is None else self.Rs * self.alpha + phi * Rs
        self.Rn = phi * Rn if self.Rn is None else self.Rn * self.alpha + phi * Rn
        if self.normalized_update:
            self.reset = False
        # do beamforming
        weight = self.weight(self.Rs, self.Rn)
        return self.beamform(do_ban(weight, Rn) if ban else weight, obs)


class MvdrBeamformer(SupervisedBeamformer):
    """
    MVDR (Minimum Variance Distortionless Response) Beamformer  (beamformer.py:515-539)
        h_mvdr(f) = R(f)_{vv}^{-1}*d(f) / [d(f)^H*R(f)_{vv}^{-1}*d(f)],  d(f) = P(R(f)_{xx})
    """

    def __init__(self, num_bins):
        super(MvdrBeamformer, self).__init__(num_bins)

    def weight(self, Rs, Rn):
        return _weights(_lib.BF_MVDR, Rs, Rn)


class MpdrBeamformer(SupervisedBeamformer):
    """
    MPDR (Minimum Power Distortionless Response) Beamformer  (beamformer.py:542-590)
        h_mpdr(f) = R(f)_{yy}^{-1}*d(f) / [d(f)^H*R(f)_{yy}^{-1}*d(f)]
    """

    def __init__(self, num_bins, whiten=False):
        super(MpdrBeamformer, self).__init__(num_bins)
        self.whiten = whiten

    def weight(self, Rs, Ry, Rn=None):
        if Rn is None:
            return _weights(_lib.BF_MPDR, Rs, None, Ry)
        return _weights(_lib.BF_MPDR_WHITEN, Rs, Rn, Ry)

    def run(self, mask_s, obs, mask_n=None, ban=False):
        Rs = self.compute_covar_mat(mask_s, obs)
        ones = torch.ones_like(mask_s) if isinstance(mask_s, torch.Tensor) else np.ones_like(mask_s)
        Ry = self.compute_covar_mat(ones, obs)
        Rn = None
        if self.whiten or ban:
            Rn = self.compute_covar_mat(1 - mask_s if mask_n is None else mask_n, obs)
        weight = self.weight(Rs, Ry, Rn=Rn if self.whiten else None)
        return self.beamform(do_ban(weight, Rn) if ban else weight, obs)


class PmwfBeamformer(SupervisedBeamformer):
    """
    PMWF (Parameterized Multichannel Non-Causal Wiener Filter)  (beamformer.py:593-659)
        h_pmwf(f) = numerator(f)*u(f) / (beta + trace(numerator(f))),
        numerator(f) = R(f)_vv^{-1}*R(f)_xx;  beta = 0 => mvdr, beta = 1 => mcwf
    """

    def __init__(self, num_bins, beta=0, ref_channel=-1, rank1_appro=""):
        super(PmwfBeamformer, self).__init__(num_bins)
        self.ref_channel = ref_channel
        self.rank1_appro = rank1_appro
        self.beta = beta

    def weight(self, Rs, Rn):
        N = Rs.shape[-1]
        if self.ref_channel >= N:
            raise RuntimeError("Reference channel ID exceeds total " +
                               f"channels: {self.ref_channel} vs {N}")
        r1 = {"eig": _lib.RANK1_EIG, "gev": _lib.RANK1_GEV}.get(self.rank1_appro, _lib.RANK1_NONE)
        return _weights(_lib.BF_PMWF, Rs, Rn, beta=float(self.beta),
                        ref_channel=int(self.ref_channel), rank1=r1)


class GevdBeamformer(SupervisedBeamformer):
    """
    Max-SNR/GEV (Generalized Eigenvalue Decomposition) Beamformer  (beamformer.py:662-682)
        h_gevd(f) = P(R(f)_xx, R(f)_vv)   P: max generalized eigenvector
    """

    def __init__(self, num_bins):
        super(GevdBeamformer, self).__init__(num_bins)

    def weight(self, Rs, Rn):
        return _weights(_lib.BF_GEVD, Rs, Rn)


class OnlineGevdBeamformer(OnlineSupervisedBeamformer):
    """
    Online version of GEVD beamformer  (beamformer.py:685-703)
    """

    def __init__(self, num_bins, num_channels, alpha=0.8):
        super(OnlineGevdBeamformer, self).__init__(num_bins, num_channels, alpha=alpha)

    def weight(self, Rs, Rn):
        return _weights(_lib.BF_GEVD, Rs, Rn)


class OnlineMvdrBeamformer(OnlineSupervisedBeamformer):
    """
    Online version of MVDR beamformer  (beamformer.py:706-728)
    """

    def __init__(self, num_bins, num_channels, alpha=0.8):
        super(OnlineMvdrBeamformer, self).__init__(num_bins, num_channels, alpha=alpha)

    def weight(self, Rs, Rn):
        return _weights(_lib.BF_MVDR, Rs, Rn)


# ---------------------------------------------------------------------------
# geometry-based beamformers (beamformer.py:106-212, 323-512)
# ---------------------------------------------------------------------------
def beam_pattern(weight, steer_vector):
    """
    Beam pattern of a fixed beamformer (beamformer.py:106-130).
        weight: B x F x N or F x N;  steer_vector: F x D x N
    returns F x D (or a list of them, one per beam)
    """
    weight, steer_vector = np.asarray(weight), np.asarray(steer_vector)
    if weight.shape[-1] != steer_vector.shape[-1] or weight.shape[-2] != steer_vector.shape[0]:
        raise RuntimeError("Shape mismatch between weight and steer_vector")

    def single_beam(w, sv):
        return np.squeeze(np.abs(sv @ np.expand_dims(w.conj(), -1)))

    if weight.ndim == 2:
        return single_beam(weight, steer_vector)
    elif weight.ndim == 3:
        return [single_beam(w, steer_vector) for w in weight]
    raise RuntimeError(f"Expect 2/3D beam weights, got {weight.ndim}")


def diffuse_covar(num_bins, dist_mat, sr=16000, c=340, diag_eps=0.1):
    """Covariance of the spherically isotropic noise field, F x N x N (beamformer.py:133-152)."""
    N, _ = dist_mat.shape
    omega = np.pi * np.arange(num_bins) * sr / (num_bins - 1)
    return np.sinc(dist_mat[None] * omega[:, None, None] / c) + np.eye(N) * diag_eps


def plane_steer_vector(distance, num_bins, c=340, sr=16000):
    """Steer vector F x N for projected distances on the DoA (beamformer.py:155-167)."""
    omega = np.pi * np.arange(num_bins) * sr / (num_bins - 1)
    return np.exp(-1j * np.outer(omega, np.asarray(distance) / c))


def linear_steer_vector(topo, doa, num_bins, c=340, sr=16000):
    """Steer vector of a linear array, doa in degrees (beamformer.py:170-186)."""
    return plane_steer_vector(np.cos(doa * np.pi / 180) * np.asarray(topo), num_bins, c=c, sr=sr)


def circular_steer_vector(redius, num_arounded, doa, num_bins, c=349, sr=16000, center=False):
    """Steer vector of a circular array (optionally with a centre microphone), beamformer.py:189-212."""
    dirc = np.arange(num_arounded) * 2 * np.pi / num_arounded
    dist = np.cos(dirc - doa * np.pi / 180) * redius
    if center:
        dist = np.concatenate([np.array([0]), dist])
    return plane_steer_vector(-dist, num_bins, c=c, sr=sr)


class FixedBeamformer(Beamformer):
    """Fixed beamformer with predefined weights F x N (beamformer.py:323-340)."""

    def __init__(self, weight):
        super().__init__()
        self.weight = weight

    def run(self, obs):
        """obs N x F x T -> F x T"""
        return self.beamform(self.weight, obs)


class DSBeamformer(Beamformer):
    """Base delay-and-sum beamformer (beamformer.py:343-377)."""

    def __init__(self, num_mics):
        super().__init__()
        self.num_mics = num_mics

    def weight(self, doa, num_bins, c=340, sr=16000):
        raise NotImplementedError

    def run(self, doa, obs, c=340, sr=16000):
        """doa in degrees, obs N x F x T -> F x T"""
        if obs.shape[-3] != self.num_mics:
            raise ValueError("Shape of obs do not match with number" +
                             f"of microphones, {self.num_mics} vs {obs.shape[-3]}")
        weight = self.weight(doa, obs.shape[-2], c=c, sr=sr)
        return self.beamform(weight, obs)


class LinearDSBeamformer(DSBeamformer):
    """Delay and sum beamformer for a linear array (beamformer.py:380-398)."""

    def __init__(self, linear_topo):
        super().__init__(len(linear_topo))
        self.linear_topo = np.array(linear_topo)

    def weight(self, doa, num_bins, c=340, sr=16000):
        return linear_steer_vector(self.linear_topo, doa, num_bins, c=c, sr=sr) / self.num_mics


class CircularDSBeamformer(DSBeamformer):
    """Delay and sum beamformer for a circular array (beamformer.py:401-428)."""

    def __init__(self, radius, num_arounded, center=False):
        super().__init__(num_arounded + 1 if center else num_arounded)
        self.radius = radius
        self.center = center
        self.num_arounded = num_arounded

    def weight(self, doa, num_bins, c=340, sr=16000):
        sv = circular_steer_vector(self.radius, self.num_arounded, doa, num_bins, c=c, sr=sr,
                                   center=self.center)
        return sv / self.num_mics


def _superdirective(steer_vector, Rn):
    """w = Rn^-1 d / (d^H Rn^-1 d) per bin (beamformer.py:453-456, 508-512)."""
    numerator = np.linalg.solve(Rn, steer_vector[..., None])[..., 0]    # stack-of-vectors semantics
    denominator = np.einsum("...d,...d->...", steer_vector.conj(), numerator)
    return numerator / np.expand_dims(denominator, axis=-1)


class LinearSDBeamformer(LinearDSBeamformer):
    """Linear super-directive beamformer in a diffuse noise field (beamformer.py:431-456)."""

    def __init__(self, linear_topo):
        super().__init__(linear_topo)
        mat = np.tile(self.linear_topo, (self.num_mics, 1))
        self.distance_mat = np.abs(mat - np.transpose(mat))

    def weight(self, doa, num_bins, c=340, sr=16000, diag_eps=0.1):
        steer_vector = super().weight(doa, num_bins, c=c, sr=sr)
        Rn = diffuse_covar(num_bins, self.distance_mat, sr=sr, c=c, diag_eps=diag_eps)
        return _superdirective(steer_vector, Rn)


class CircularSDBeamformer(CircularDSBeamformer):
    """Circular super-directive beamformer in a diffuse noise field (beamformer.py:459-512)."""

    def __init__(self, radius, num_arounded, center=False):
        super().__init__(radius, num_arounded, center=center)
        self.distance_mat = self._compute_distance_mat()

    def _compute_distance_mat(self):
        distance_mat = np.zeros((self.num_mics, self.num_mics))
        raw = 0
        if self.center:
            distance_mat[0, 1:] = self.radius
            raw = 1
        ang = np.pi / self.num_arounded
        for r in range(raw, self.num_mics):
            for c in range(r + 1, self.num_mics):
                distance_mat[r, c] = np.abs(np.sin((c - r) * ang) * 2 * self.radius)
        distance_mat += distance_mat.T
        return distance_mat

    def weight(self, doa, num_bins, c=340, sr=16000, diag_eps=1e-5):
        steer_vector = super().weight(doa, num_bins, c=c, sr=sr)
        Rn = diffuse_covar(num_bins, self.distance_mat, sr=sr, c=c, diag_eps=diag_eps)
        return _superdirective(steer_vector, Rn)
