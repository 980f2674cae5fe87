"""
The per-bin fp64 weight solves (setk_weights, setk_ban, setk_rank1) against a
40-digit restatement of oracle/beamformer_oracle.py, on Hermitian matrices with
a prescribed spectrum.  The same functions run

  * in the CPU tier against tests/emu/libsetk_b200_emu.so at a few shapes, and
  * in the GPU tier against libsetk_b200.so on an H100, over every route.

Reference.  mpmath at DPS digits, on the exact values the kernel receives (after
complex64 rounding), read the way the kernel reads them: the lower triangle,
Hermitised, for the eigen and Cholesky steps (principal_eigvec, gev_principal,
load_lower_hermitian), the full matrix for LU (np.linalg.solve).  It keeps the
library's conventions: the principal vector has unit norm and a real,
non-negative component 0; BAN, rank-1 and the PMWF SNR keep their EPSILON
floors; a Cholesky that fails is retried on Rn + tr/C * {1e-10, 1e-8, ..., 1e-2} I.

Tolerance model, one for every route:  err <= K_TOL * C * u * cond, with
  u     2^-53 for the fp64 arithmetic, plus 2^-24 when the output is complex64;
  cond  the first-order condition number of the quantity:
          principal eigenvector of R       ||R|| / gap
          MVDR, MPDR                       kappa(D) + ||Rs|| / gap(Rs)   (D = Rn or Ry)
          GEVD, PEVD with Rn               kappa(Rn) * (1 + |mu|max / gap(mu))   (mu: the pencil)
          PMWF                             kappa(Rn), plus the rank-1 vector's when it has one
          BAN                              the component-wise condition of w^H Rn w and w^H Rn^2 w;
        Weights that inherit a canonical vector's phase (component 0 real, >= 0: PEVD, MVDR, MPDR,
        MPDR-whiten, GEVD and their BAN) are compared as they are, with cond times that vector's
        phase factor 1 + max|v| / |v_0|; only where v_0 = 0 (a dead channel 0) is the phase
        aligned first;
  err   max |w - w_ref| / max |w_ref| per bin.
WORST records the largest err / bound per route and dtype; each test module clears it first and
prints it after its last test.
"""
import zlib

import mpmath
import numpy as np
import torch

from oracle.stft_oracle import EPSILON
from setk_b200 import _lib
from setk_b200 import plan as P

DPS = 40
K_TOL = 32.0
U64 = 2.0 ** -53
U32 = 2.0 ** -24
EPS = float(EPSILON)
LOADS = [1e-10]                              # gev_principal's ladder, as the kernels compute it
for _ in range(4):
    LOADS.append(LOADS[-1] * 100.0)

KINDS = {"pevd": _lib.BF_PEVD, "pevd_rn": _lib.BF_PEVD, "mvdr": _lib.BF_MVDR, "mpdr": _lib.BF_MPDR,
         "mpdr_whiten": _lib.BF_MPDR_WHITEN, "gevd": _lib.BF_GEVD, "pmwf": _lib.BF_PMWF}

# (family, parameter): the matrices of one utterance (see make_family)
SWEEP_FAMILIES = ([("cond", c) for c in (1e1, 1e4, 1e8, 1e12)] +
                  [("gap", g) for g in (1e-1, 1e-4, 1e-7)] +
                  [("pgap", g) for g in (1e-1, 1e-4, 1e-7)] +
                  [("rank1", None), ("scale", 40), ("scale", -40)])

WORST = {}


def record(route, ratio):
    WORST[route] = max(WORST.get(route, 0.0), float(ratio))


def report():
    return "\n".join(f"  {k:<44s} worst err/bound {v:.3e}" for k, v in sorted(WORST.items()))


def bound(C, cond, out_c64):
    return K_TOL * C * (U64 + (U32 if out_c64 else 0.0)) * cond


# ----------------------------------------------------------------------------
# generators
# ----------------------------------------------------------------------------
def haar_unitary(rng, C):
    """Random unitary from a QR with the phases of R's diagonal fixed (Haar distributed)."""
    Z = rng.standard_normal((C, C)) + 1j * rng.standard_normal((C, C))
    Q, R = np.linalg.qr(Z)
    d = np.diag(R)
    return Q * (d / np.abs(d))[None, :]


def hermitian(Q, lam):
    """Q diag(lam) Q^H, exactly Hermitian with a real diagonal."""
    R = (Q * np.asarray(lam, dtype=np.float64)[None, :]) @ np.conj(Q.T)
    R = (R + np.conj(R.T)) / 2
    R[np.diag_indices(len(lam))] = R.diagonal().real
    return R


def spectrum_cond(C, cond):
    """C eigenvalues from 1 down to 1/cond, geometric."""
    return np.array([1.0]) if C == 1 else cond ** (-np.arange(C) / (C - 1))


def spectrum_gap(C, gap):
    """Top two eigenvalues 1 and 1 - gap (relative gap `gap`), the rest below 1/2, down to 1e-3."""
    if C == 1:
        return np.array([1.0])
    rest = 0.5 * (2e-3) ** (np.arange(C - 2) / max(C - 3, 1))
    return np.concatenate([[1.0, 1.0 - gap], rest[:C - 2]])


def dyadic_vector(rng, C):
    """A vector of small integers: s s^H is exact in complex64, so Rs is exactly rank 1."""
    s = rng.integers(-8, 9, C) + 1j * rng.integers(-8, 9, C)
    s[0] += 9
    return s.astype(np.complex128)


def make_bin(rng, family, param, C):
    """One (Rs, Rn) pair of a family, complex128, exactly Hermitian."""
    Rn = hermitian(haar_unitary(rng, C), spectrum_cond(C, 1e2))
    Rs = hermitian(haar_unitary(rng, C), spectrum_gap(C, 1e-1))
    if family == "cond":                   # cond(Rn) = param
        Rn = hermitian(haar_unitary(rng, C), spectrum_cond(C, param))
    elif family == "gap":                  # relative gap of Rs's top two eigenvalues = param
        Rs = hermitian(haar_unitary(rng, C), spectrum_gap(C, param))
    elif family == "pgap":                 # relative gap of the pencil (Rs, Rn) = param
        L = np.linalg.cholesky(Rn)
        Rs = L @ hermitian(haar_unitary(rng, C), spectrum_gap(C, param)) @ np.conj(L.T)
        Rs = (Rs + np.conj(Rs.T)) / 2
        Rs[np.diag_indices(C)] = Rs.diagonal().real
    elif family == "rank1":                # a single source
        s = dyadic_vector(rng, C)
        Rs = np.outer(s, np.conj(s))
    elif family == "silent":               # a silent bin
        Rs = np.zeros((C, C), dtype=np.complex128)
    elif family == "rankdef":              # fewer noise frames than channels: X X^H, X C x k, k < C
        k = max(1, C // 2)
        X = rng.standard_normal((C, k)) + 1j * rng.standard_normal((C, k))
        Rn = X @ np.conj(X.T) / k
        Rn = (Rn + np.conj(Rn.T)) / 2
        Rn[np.diag_indices(C)] = Rn.diagonal().real
    elif family == "dead":                 # microphone `param` silent: its row and column are zero
        Rs[param, :] = 0
        Rs[:, param] = 0
        Rn[param, :] = 0
        Rn[:, param] = 0
    elif family == "indef":                # one eigenvalue of Rn at -3e-3 tr/C: only the last rung is PD
        lam = spectrum_cond(C, 1e1)
        lam[-1] = -3e-3 * lam[:-1].sum() / (C + 3e-3)          # = -3e-3 * tr / C
        Rn = hermitian(haar_unitary(rng, C), lam)
    elif family == "scale":                # a power-of-two scaled copy of a generic pair
        Rs, Rn = Rs * 2.0 ** param, Rn * 2.0 ** param
    else:
        raise ValueError(family)
    return Rs, Rn


def make_family(seed, family, param, C, F):
    """(Rs, Rn) stacks (F, C, C) of one family, complex128."""
    rng = np.random.default_rng([seed, C, F, zlib.crc32(f"{family} {param}".encode())])
    pairs = [make_bin(rng, family, param, C) for _ in range(F)]
    return np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])


# ----------------------------------------------------------------------------
# the 40-digit reference
# ----------------------------------------------------------------------------
def lower_hermitian(A):
    """The Hermitian matrix the kernels read from A's lower triangle (numpy, exact)."""
    L = np.tril(A, -1)
    H = L + np.conj(L.T)
    H[np.diag_indices(A.shape[0])] = A.diagonal().real
    return H


def to_mp(A):
    A = np.asarray(A, dtype=np.complex128)
    if A.ndim == 1:
        return [mpmath.mpc(float(z.real), float(z.imag)) for z in A]
    M = mpmath.matrix(A.shape[0], A.shape[1])
    for i in range(A.shape[0]):
        for j in range(A.shape[1]):
            M[i, j] = mpmath.mpc(float(A[i, j].real), float(A[i, j].imag))
    return M


def to_np(v):
    return np.array([complex(z) for z in v], dtype=np.complex128)


def phase_factor(v):
    """1 + max|v| / |v_0| for the canonical vector v: how much its component-0 phase rule amplifies
    an error in v.  None when v_0 = 0, where the rule leaves the phase to the rounding."""
    m0 = abs(v[0])
    return 1.0 + float(max(abs(z) for z in v) / m0) if m0 > 0 else None


def with_phase(cond, pf):
    """(cond, align) of a quantity that inherits a canonical vector's phase."""
    return (cond, True) if pf is None else (cond * pf, False)


def mp_principal(H):
    """Principal eigenvector of the Hermitian mp matrix H, library phase convention.
    Returns (vector, eigenvalues ascending)."""
    C = H.rows
    E, Q = mpmath.eighe(H)
    v = [Q[i, C - 1] for i in range(C)]
    n = mpmath.sqrt(mpmath.fsum(abs(z) ** 2 for z in v))
    m0 = abs(v[0])
    ph = mpmath.conj(v[0]) / m0 if m0 > 0 else mpmath.mpf(1)
    v = [z * ph / n for z in v]
    if m0 > 0:
        v[0] = mpmath.mpc(v[0].real, 0)
    return v, [E[i] for i in range(C)]


def mp_cholesky(H):
    """Lower Cholesky factor of a Hermitian mp matrix, or None if a pivot is not positive."""
    C = H.rows
    L = mpmath.matrix(C, C)
    for j in range(C):
        d = H[j, j].real - mpmath.fsum(abs(L[j, k]) ** 2 for k in range(j))
        if not d > 0:
            return None
        L[j, j] = mpmath.sqrt(d)
        for i in range(j + 1, C):
            s = H[i, j] - mpmath.fsum(L[i, k] * mpmath.conj(L[j, k]) for k in range(j))
            L[i, j] = s / L[j, j]
    return L


def mp_solve(A, B):
    """A^-1 B for an mp matrix A and a list of right-hand sides (lists), Gaussian elimination
    with partial pivoting.  None when A is exactly singular."""
    C = A.rows
    M = [[A[i, j] for j in range(C)] + [b[i] for b in B] for i in range(C)]
    n = C + len(B)
    for k in range(C):
        p = max(range(k, C), key=lambda i: abs(M[i][k]))
        if M[p][k] == 0:
            return None
        M[k], M[p] = M[p], M[k]
        for i in range(k + 1, C):
            f = M[i][k] / M[k][k]
            if f != 0:
                M[i] = [M[i][j] - f * M[k][j] if j >= k else M[i][j] for j in range(n)]
    X = [[mpmath.mpc(0)] * C for _ in B]
    for r in range(len(B)):
        for i in range(C - 1, -1, -1):
            s = M[i][C + r] - mpmath.fsum(M[i][k] * X[r][k] for k in range(i + 1, C))
            X[r][i] = s / M[i][i]
    return X


def matvec(A, v):
    return [mpmath.fsum(A[i, j] * v[j] for j in range(A.cols)) for i in range(A.rows)]


def dotc(a, b):
    return mpmath.fsum(mpmath.conj(x) * y for x, y in zip(a, b))


def kernel_trace(Rn):
    """tr(Rn) as the one-thread kernel sums it (fp64, in order)."""
    tr = 0.0
    for i in range(Rn.shape[0]):
        tr += float(Rn[i, i].real)
    return tr


def loaded(Rn, load):
    """Rn's diagonal plus load * tr / C, rounded as gev_principal does."""
    C = Rn.shape[0]
    add = load * kernel_trace(Rn) / C
    R = Rn.copy()
    for i in range(C):
        R[i, i] = complex(R[i, i].real + add, R[i, i].imag)
    return R


def kappa(A):
    s = np.linalg.svd(A, compute_uv=False)
    return float(s[0] / s[-1]) if s[-1] > 0 else np.inf


def _mp(fn):
    """Run a reference method at DPS digits."""
    def wrapped(*args, **kw):
        with mpmath.workdps(DPS):
            return fn(*args, **kw)
    return wrapped


class BinRef:
    """Reference quantities of one bin, computed on demand: Rs, Rn, Ry exactly as the kernel
    receives them (complex128 copies of the possibly complex64 inputs)."""

    def __init__(self, Rs, Rn=None, Ry=None):
        self.Rs = np.asarray(Rs, dtype=np.complex128)
        self.Rn = None if Rn is None else np.asarray(Rn, dtype=np.complex128)
        self.Ry = None if Ry is None else np.asarray(Ry, dtype=np.complex128)
        self.C = self.Rs.shape[0]
        self._eig = None
        self._gev = {}
        self._memo = {}

    @_mp
    def eig(self):
        """(principal eigenvector of Rs, cond, phase factor) -- cond inf when the top eigenvalue is
        multiple."""
        if self._eig is None:
            v, E = mp_principal(to_mp(lower_hermitian(self.Rs)))
            C = self.C
            top = max(abs(E[0]), abs(E[-1]))
            gap = E[-1] - E[-2] if C > 1 else top
            cond = 1.0 if C == 1 else (float(top / gap) if gap > 0 else np.inf)
            self._eig = (v, cond, phase_factor(v))
        return self._eig

    @_mp
    def gev(self, load=None):
        """(w, cond, load used, phase factor of y) of gev_principal: w = L^-H y, y the principal eigenvector of
        L^-1 Rs L^-H with Rn (+ the ladder's loading) = L L^H.  `load` None: the ladder, with PD
        decided exactly; otherwise that rung.  w None if no rung is positive definite."""
        if load not in self._gev:
            Hn = lower_hermitian(self.Rn)
            rungs = [0.0] + LOADS if load is None else [load]
            L = None
            for ld in rungs:
                Rl = loaded(Hn, ld) if ld else Hn
                L = mp_cholesky(to_mp(Rl))
                if L is not None:
                    break
            if L is None:
                self._gev[load] = (None, np.inf, None, None)
                return self._gev[load]
            C = self.C
            Hs = to_mp(lower_hermitian(self.Rs))
            Li = mpmath.inverse(L)
            M = Li * Hs * Li.H
            M = (M + M.H) / 2
            y, mu = mp_principal(M)
            w = [mpmath.mpc(0)] * C                                  # L^H w = y
            for i in range(C - 1, -1, -1):
                s = y[i] - mpmath.fsum(mpmath.conj(L[k, i]) * w[k] for k in range(i + 1, C))
                w[i] = s / L[i, i]
            top = max(abs(mu[0]), abs(mu[-1]))
            gap = mu[-1] - mu[-2] if C > 1 else top
            cg = 1.0 if C == 1 else (float(top / gap) if gap > 0 else np.inf)
            self._gev[load] = (w, kappa(Rl) * (1.0 + cg), ld, phase_factor(y))
        return self._gev[load]

    # -- the beamformers (oracle/beamformer_oracle.py, evaluated exactly) -------------
    # Each returns (w, cond, align).  The weights carry the phase of a canonical vector (component 0
    # real, >= 0), so they are compared as they are, with cond widened by that vector's phase
    # factor; only where its component 0 is zero (a dead channel 0) is the phase aligned first.
    def pevd(self):
        v, cond, pf = self.eig()
        return (to_np(v),) + with_phase(cond, pf)

    def gevd(self, load=None):
        w, cond, _, pf = self.gev(load)
        return (None if w is None else to_np(w),) + with_phase(cond, pf)

    @_mp
    def _distortionless(self, D, d, cond_d, pf):
        Dm = to_mp(D)
        x = mp_solve(Dm, [d])
        if x is None:
            return None, np.inf, False
        n = x[0]
        den = dotc(d, n)
        return (to_np([z / den for z in n]),) + with_phase(kappa(D) + cond_d, pf)

    def mvdr(self):
        d, cd, pf = self.eig()
        return self._distortionless(self.Rn, d, cd, pf)

    def mpdr(self):
        d, cd, pf = self.eig()
        return self._distortionless(self.Ry, d, cd, pf)

    def mpdr_whiten(self):
        g, cg, _, pf = self.gev()
        if g is None:
            return None, np.inf, False
        d = matvec(to_mp(self.Rn), g)
        return self._distortionless(self.Ry, d, kappa(self.Rn) * cg, pf)

    def rank1(self, gev):
        key = ("rank1", gev)
        if key not in self._memo:
            self._memo[key] = self._rank1(gev)
        return self._memo[key]

    def pmwf_matrix(self, beta, rank1=""):
        key = ("pmwf", beta, rank1)
        if key not in self._memo:
            self._memo[key] = self._pmwf_matrix(beta, rank1)
        return self._memo[key]

    @_mp
    def _rank1(self, gev):
        """rank1_constraint(Rs, Rn if gev): (R1 (C, C), cond)."""
        if gev:
            g, cg, _, _ = self.gev()
            if g is None:
                return None, np.inf
            p, cond = matvec(to_mp(self.Rn), g), kappa(self.Rn) * cg
        else:
            p, cond, _ = self.eig()
        tr = mpmath.fsum(to_mp(self.Rs)[i, i].real for i in range(self.C))
        tr1 = mpmath.fsum(abs(z) ** 2 for z in p)
        scale = tr / max(tr1, mpmath.mpf(EPS))
        R1 = np.array([[complex(scale * p[i] * mpmath.conj(p[j])) for j in range(self.C)]
                       for i in range(self.C)])
        return R1, cond

    @_mp
    def _pmwf_matrix(self, beta, rank1):
        """W = Rn^-1 Rs' / (beta + tr(Rn^-1 Rs')), Rs' Rs or its rank-1 model: (W (C, C), cond, Rs')."""
        C = self.C
        if rank1:
            R1, cond1 = self.rank1(rank1 == "gev")
            if R1 is None:
                return None, np.inf, None
        else:
            R1, cond1 = self.Rs, 0.0
        Rs = to_mp(R1)
        X = mp_solve(to_mp(self.Rn), [[Rs[i, c] for i in range(C)] for c in range(C)])
        if X is None:
            return None, np.inf, None
        den = beta + mpmath.fsum(X[c][c] for c in range(C))
        W = np.array([[complex(X[c][i] / den) for c in range(C)] for i in range(C)])
        G = np.array([[complex(X[c][i]) for c in range(C)] for i in range(C)])
        kn = kappa(self.Rn)
        cond = kn * (1.0 + np.abs(G).max() * C / max(abs(complex(den)), 1e-300)) + kn * cond1
        return W, cond, R1

    @_mp
    def ban(self, w, cond_w=0.0):
        """do_ban(w, Rn) on the given w: (w', cond)."""
        Rn = to_mp(self.Rn)
        wm = to_mp(w)
        u = matvec(Rn, wm)
        v = matvec(Rn, u)
        num, den = dotc(wm, v), dotc(wm, u)
        g = mpmath.sqrt(abs(num)) / max(den.real, mpmath.mpf(EPS))
        aw, aR = np.abs(w), np.abs(self.Rn)
        cnum = float(aw @ aR @ aR @ aw) / max(abs(complex(num)), 1e-300)
        cden = float(aw @ aR @ aw) / max(float(den.real), 1e-300) if den.real > EPS else 0.0
        return to_np([z * g for z in wm]), cond_w + cnum + cden


# ----------------------------------------------------------------------------
# comparisons
# ----------------------------------------------------------------------------
def err_vec(w, ref, align=True):
    w = np.asarray(w, dtype=np.complex128)
    if align:
        inner = np.sum(ref * np.conj(w))
        if abs(inner) > 0:
            w = w * (inner / abs(inner))
    return float(np.max(np.abs(w - ref)) / max(np.max(np.abs(ref)), 1e-300))


def check(route, C, w, ref, cond, out_c64, align=False, what=""):
    """Assert one bin's err <= bound and record err / bound under `route`."""
    if ref is None or not np.isfinite(cond):
        return
    err = err_vec(w, ref, align)
    b = bound(C, cond, out_c64)
    record(route, err / b)
    assert err <= b, f"{route} {what}: err {err:.3e} > bound {b:.3e} (cond {cond:.3e})"


def tensors(device, dtype, *mats):
    return [None if m is None else torch.from_numpy(np.ascontiguousarray(m.astype(dtype))).to(device)
            for m in mats]


def _route(C, kind, rn=False):
    """Which weights kernel runs (weights.cu / weights_coop.cu dispatch)."""
    if kind in ("pmwf", "mpdr_whiten") or C < 4:
        return "thread"
    if C == 4:
        return "coop4" if kind in ("mvdr", "mpdr") or (kind == "pevd" and not rn) else "thread"
    return "coop"


# ----------------------------------------------------------------------------
# the accuracy sweep
# ----------------------------------------------------------------------------
def build_batch(seed, C, F, families):
    """Rs, Rn, Ry stacks (B, F, C, C), one utterance per family."""
    Rs, Rn = zip(*[make_family(seed, f, p, C, F) for f, p in families])
    Rs, Rn = np.stack(Rs), np.stack(Rn)
    return Rs, Rn, Rs + Rn


def check_sweep(device, C, F, families, in_dtype, seed=0, kinds=None, pmwf=True, ban=True):
    """Every kind on `families` (one utterance each) in `in_dtype`, outputs in complex128 and
    complex64, against the reference.  Also: no error bit on any of these inputs."""
    Rs, Rn, Ry = build_batch(seed, C, F, families)
    B = Rs.shape[0]
    Rs_k, Rn_k, Ry_k = (m.astype(in_dtype).astype(np.complex128) for m in (Rs, Rn, Ry))
    tRs, tRn, tRy = tensors(device, in_dtype, Rs, Rn, Ry)
    refs = [[BinRef(Rs_k[b, f], Rn_k[b, f], Ry_k[b, f]) for f in range(F)] for b in range(B)]
    tag = "c64" if in_dtype == np.complex64 else "c128"
    kinds = ["pevd", "pevd_rn", "mvdr", "mpdr", "mpdr_whiten", "gevd"] if kinds is None else kinds

    def run(kind, out, **kw):
        rn = tRn if kind not in ("pevd", "mpdr") else None
        ry = tRy if kind in ("mpdr", "mpdr_whiten") else None
        w, st, used = P.weights(KINDS[kind], tRs, rn, ry, out_dtype=out, **kw)
        st = st.cpu().numpy()
        assert not np.any(st & _lib.ST_ERROR_MASK), (kind, C, tag, st)
        assert not np.any(st & _lib.ST_NO_CONVERGE)
        if in_dtype == np.complex128:       # every Rn here is PD; its complex64 rounding need not be
            assert not np.any(st & _lib.ST_REGULARIZED), (kind, st)
        return w.cpu().numpy(), used.cpu().numpy()

    for out in (torch.complex128, torch.complex64):
        oc = out == torch.complex64
        otag = f"{tag}->{'c64' if oc else 'c128'}"
        for kind in kinds:
            w, _ = run(kind, out)
            route = f"{kind} C={C} {_route(C, kind, kind == 'pevd_rn')} {otag}"
            for b in range(B):
                for f in range(F):
                    r = refs[b][f]
                    ref, cond, al = {"pevd": r.pevd, "pevd_rn": r.gevd, "mvdr": r.mvdr, "mpdr": r.mpdr,
                                 "mpdr_whiten": r.mpdr_whiten, "gevd": r.gevd}[kind]()
                    check(route, C, w[b, f], ref, cond, oc, align=al, what=f"{families[b]} bin {f}")
                    if kind == "pevd" and ref is not None and np.isfinite(cond) and not oc:
                        assert w[b, f, 0].imag == 0 and w[b, f, 0].real >= 0      # the phase convention
                        assert abs(np.linalg.norm(w[b, f]) - 1) <= 8 * C * U64
            if ban and kind in ("mvdr", "gevd"):
                wb, _ = run(kind, out, ban=True)
                for b in range(B):
                    for f in range(F):
                        r = refs[b][f]
                        ref, cond, al = r.mvdr() if kind == "mvdr" else r.gevd()
                        if ref is None or not np.isfinite(cond):
                            continue
                        ref_b, cond_b = r.ban(ref, cond)
                        check(f"{kind}+ban C={C} {_route(C, kind)} {otag}", C,
                              wb[b, f], ref_b, cond_b, oc, align=al, what=f"{families[b]} bin {f}")
        if not pmwf:
            continue
        for beta in (0.0, 1.0):
            for r1 in ("", "eig", "gev"):
                code = {"": _lib.RANK1_NONE, "eig": _lib.RANK1_EIG, "gev": _lib.RANK1_GEV}[r1]
                for ref_ch in (-1, C - 1):
                    w, used = run("pmwf", out, beta=beta, ref_channel=ref_ch, rank1=code)
                    route = f"pmwf{'+' + r1 if r1 else ''} C={C} thread {otag}"
                    Ws = [[refs[b][f].pmwf_matrix(beta, r1) for f in range(F)] for b in range(B)]
                    for b in range(B):
                        if ref_ch < 0:
                            check_pmwf_ref(Ws[b], Rn_k[b], int(used[b]))
                        ch = ref_ch if ref_ch >= 0 else int(used[b])
                        for f in range(F):
                            W, cond, _ = Ws[b][f]
                            check(route, C, w[b, f], None if W is None else W[:, ch], cond, oc,
                                  align=False, what=f"{families[b]} bin {f} beta {beta} ref {ref_ch}")


def check_pmwf_ref(Ws, Rn, used):
    """The automatic reference channel: argmax_c of sum_f w_c^H Rs' w_c / max(EPS, sum_f w_c^H Rn w_c)
    (pmwf_snr, Rs' the rank-1 model when there is one).  The kernel's choice must be the
    reference's, or tie with it to 1e-9."""
    if any(W is None for W, _, _ in Ws):
        return
    C = Rn.shape[-1]
    snr = []
    for c in range(C):
        ps = sum((np.conj(W[:, c]) @ R1 @ W[:, c]).real for W, _, R1 in Ws)
        pn = sum((np.conj(W[:, c]) @ Rn[f] @ W[:, c]).real for f, (W, _, _) in enumerate(Ws))
        snr.append(ps / max(EPS, pn))
    best = int(np.argmax(snr))
    assert used == best or snr[used] >= snr[best] * (1 - 1e-9), (used, best, snr)


def check_post(device, C, F, families, in_dtype, seed=1):
    """setk_ban and setk_rank1 (plan.ban / plan.rank1) against the reference."""
    Rs, Rn, _ = build_batch(seed, C, F, families)
    B = Rs.shape[0]
    rng = np.random.default_rng([seed, C, 7])
    w = rng.standard_normal((B, F, C)) + 1j * rng.standard_normal((B, F, C))
    Rs_k, Rn_k, w_k = (m.astype(in_dtype).astype(np.complex128) for m in (Rs, Rn, w))
    tRs, tRn, tw = tensors(device, in_dtype, Rs, Rn, w)
    oc = in_dtype == np.complex64
    tag = "c64" if oc else "c128"
    out = P.ban(tw, tRn).cpu().numpy()
    for b in range(B):
        for f in range(F):
            ref, cond = BinRef(Rs_k[b, f], Rn_k[b, f]).ban(w_k[b, f])
            check(f"setk_ban C={C} {tag}", C, out[b, f], ref, cond, oc, align=False,
                  what=f"{families[b]} bin {f}")
    for gev in (False, True):
        R1, st = P.rank1(tRs, tRn if gev else None)
        st = st.cpu().numpy()
        assert not np.any(st & _lib.ST_ERROR_MASK), st
        if in_dtype == np.complex128:
            assert not np.any(st & _lib.ST_REGULARIZED), st
        R1 = R1.cpu().numpy()
        for b in range(B):
            for f in range(F):
                ref, cond = BinRef(Rs_k[b, f], Rn_k[b, f]).rank1(gev)
                if ref is None:
                    continue
                check(f"setk_rank1 {'gev' if gev else 'eig'} C={C} {tag}", C, R1[b, f].ravel(),
                      ref.ravel(), cond, oc, align=False, what=f"{families[b]} bin {f}")


# ----------------------------------------------------------------------------
# the status contract
# ----------------------------------------------------------------------------
def check_dead_channel(device, C, F=3, dead=None, seed=2):
    """A dead microphone in utterance 1 of 3.
    GEVD / PEVD with Rn: attempt 0 meets an exact zero pivot, attempt 1 (load 1e-10 tr/C) succeeds:
    ST_REGULARIZED only, weights = the reference's at that load.
    MVDR / MPDR: ST_SINGULAR for that utterance only (the reference's per-utterance LinAlgError)."""
    dead = C // 2 if dead is None else dead
    fams = [("cond", 1e2), ("dead", dead), ("cond", 1e2)]
    Rs, Rn, Ry = build_batch(seed, C, F, fams)
    tRs, tRn, tRy = tensors(device, np.complex128, Rs, Rn, Ry)
    for kind in ("gevd", "pevd_rn"):
        w, st, _ = P.weights(KINDS[kind], tRs, tRn)
        st, w = st.cpu().numpy(), w.cpu().numpy()
        assert st[0] == 0 and st[2] == 0, st
        assert st[1] == _lib.ST_REGULARIZED, st
        for f in range(F):
            ref, cond, al = BinRef(Rs[1, f], Rn[1, f]).gevd(load=LOADS[0])
            check(f"{kind} dead channel C={C} {_route(C, 'gevd')}", C, w[1, f], ref, cond, False, align=al)
    for kind, D in (("mvdr", tRn), ("mpdr", tRy)):
        w, st, _ = P.weights(KINDS[kind], tRs, tRn if kind == "mvdr" else None, D if kind == "mpdr" else None)
        st = st.cpu().numpy()
        assert st[0] == 0 and st[2] == 0, (kind, st)
        assert st[1] & _lib.ST_SINGULAR, (kind, st)


def check_silent(device, C, F=2, seed=8):
    """Rs = 0.  Its principal vector is not unique, so the eigenvector kinds only owe finite
    weights and no error bit; PMWF with beta 1 and the rank-1 model owe exact zeros, and PMWF with
    beta 0 divides 0 by 0 like the reference and reports it."""
    Rs, Rn, Ry = build_batch(seed, C, F, [("silent", None)])
    tRs, tRn, tRy = tensors(device, np.complex128, Rs, Rn, Ry)
    for kind in ("pevd", "pevd_rn", "mvdr", "mpdr", "mpdr_whiten", "gevd"):
        rn = tRn if kind not in ("pevd", "mpdr") else None
        ry = tRy if kind in ("mpdr", "mpdr_whiten") else None
        w, st, _ = P.weights(KINDS[kind], tRs, rn, ry)
        assert int(st[0]) == 0, (kind, int(st[0]))
        assert np.all(np.isfinite(w.cpu().numpy()))
    w, st, _ = P.weights(_lib.BF_PMWF, tRs, tRn, beta=1.0, ref_channel=0)
    assert int(st[0]) == 0 and not w.cpu().numpy().any()
    w, st, _ = P.weights(_lib.BF_PMWF, tRs, tRn, beta=0.0, ref_channel=0)
    assert int(st[0]) == _lib.ST_NONFINITE
    for rn in (None, tRn):
        R1, st = P.rank1(tRs, rn)
        assert int(st[0]) == 0 and not R1.cpu().numpy().any()


def check_ladder_depth(device, C, F=3, seed=3):
    """Rn with one eigenvalue at -3e-3 tr/C: only the last rung (1e-2) is positive definite."""
    Rs, Rn, _ = build_batch(seed, C, F, [("indef", None)])
    tRs, tRn = tensors(device, np.complex128, Rs, Rn)
    w, st, _ = P.weights(_lib.BF_GEVD, tRs, tRn)
    st, w = st.cpu().numpy(), w.cpu().numpy()
    assert st[0] == _lib.ST_REGULARIZED, st
    for f in range(F):
        ref, cond, al = BinRef(Rs[0, f], Rn[0, f]).gevd(load=LOADS[-1])
        check(f"gevd ladder 1e-2 C={C} {_route(C, 'gevd')}", C, w[0, f], ref, cond, False, align=al)


def check_rank_deficient(device, C, F=4, seed=4):
    """Rn = X X^H with fewer columns than channels: whether the Cholesky fails is a matter of
    rounding, so only finite weights, no error bit, and a generalised-eigen residual at the load
    the ladder reached, as small as a backward-stable solve leaves it:
        ||Rs w - mu Rl w|| <= K_TOL * C * u * (||Rs|| + |mu| ||Rl||) ||w||,  mu = w^H Rs w / w^H Rl w,
    Rl = Rn when the status has no ST_REGULARIZED, else Rn + load * tr / C * I for one of the
    loaded rungs.  Each bin is an utterance of its own, so its status names its rung."""
    Rs, Rn, _ = build_batch(seed, C, F, [("rankdef", None)])
    Rs, Rn = Rs.reshape(F, 1, C, C), Rn.reshape(F, 1, C, C)
    tRs, tRn = tensors(device, np.complex128, Rs, Rn)
    for kind in ("gevd", "pevd_rn"):
        w, st, _ = P.weights(KINDS[kind], tRs, tRn)
        st, w = st.cpu().numpy(), w.cpu().numpy()
        assert not np.any(st & _lib.ST_ERROR_MASK), st
        assert np.all(np.isfinite(w))
        for b in range(F):
            Hs, Hn = lower_hermitian(Rs[b, 0]), lower_hermitian(Rn[b, 0])
            x = w[b, 0]
            best = np.inf
            for ld in (LOADS if st[b] & _lib.ST_REGULARIZED else [0.0]):
                Rl = loaded(Hn, ld) if ld else Hn
                mu = (np.conj(x) @ Hs @ x).real / (np.conj(x) @ Rl @ x).real
                res = np.linalg.norm(Hs @ x - mu * (Rl @ x))
                scale = (np.linalg.norm(Hs, 2) + abs(mu) * np.linalg.norm(Rl, 2)) * np.linalg.norm(x)
                best = min(best, res / scale / bound(C, 1.0, False))
            record(f"{kind} rank-deficient Rn residual C={C}", best)
            assert best <= 1.0, (kind, C, b, int(st[b]), best)


# ----------------------------------------------------------------------------
# batch-composition invariance (the thread-group routes)
# ----------------------------------------------------------------------------
NEIGHBOURS = ("target", "diagonal", "slow", "ladder", "dead")


def make_neighbour(rng, kind, C):
    if kind == "target":
        return make_bin(rng, "cond", 1e3, C)
    if kind == "diagonal":                 # Jacobi converges in 0 sweeps
        d = np.sort(rng.uniform(0.1, 1.0, C))[::-1]
        return np.diag(d).astype(np.complex128), np.diag(rng.uniform(0.1, 1.0, C)).astype(np.complex128)
    if kind == "slow":                     # many sweeps: tight gaps, ill-conditioned Rn
        Rs, _ = make_bin(rng, "gap", 1e-7, C)
        _, Rn = make_bin(rng, "cond", 1e12, C)
        return Rs, Rn
    if kind == "ladder":                   # GEVD walks the loading ladder to its last rung
        return make_bin(rng, "indef", None, C)
    return make_bin(rng, "dead", int(rng.integers(C)), C)      # NaN weights (MVDR, MPDR)


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype == np.complex128 else np.uint32)


def check_invariance(device, C, B, F, kinds, seed=5, dtype=np.complex128, out=torch.complex128):
    """Each bin's weights are bit-identical whether it is solved alone or inside a batch whose
    thread-group neighbours converge in 0 sweeps or many, walk the loading ladder, produce NaN
    weights, or are inactive (B * F not a multiple of the groups per CTA)."""
    rng = np.random.default_rng([seed, C, B, F])
    # warps alternate: targets among 0-sweep neighbours, then targets among slow, ladder and NaN
    # ones, so that groups of one warp, and whole warps, finish at very different times
    GS = 2 if C <= 2 else 4 if C <= 4 else 8 if C <= 8 else 16
    warp = np.arange(B * F).reshape(B, F) // (32 // GS)
    fast = rng.choice([0, 1], size=(B, F), p=[0.5, 0.5])
    slow = rng.choice([0, 2, 3, 4], size=(B, F), p=[0.4, 0.2, 0.2, 0.2])
    labels = np.where(warp % 2 == 0, fast, slow)
    pairs = [[make_neighbour(rng, NEIGHBOURS[labels[b, f]], C) for f in range(F)] for b in range(B)]
    Rs = np.stack([np.stack([p[0] for p in row]) for row in pairs])
    Rn = np.stack([np.stack([p[1] for p in row]) for row in pairs])
    Ry = Rs + Rn
    tRs, tRn, tRy = tensors(device, dtype, Rs, Rn, Ry)
    for kind, ban in kinds:
        rn = tRn if kind in ("mvdr", "gevd", "pevd_rn") or ban else None
        ry = tRy if kind == "mpdr" else None
        w = P.weights(KINDS[kind], tRs, rn, ry, ban=ban, out_dtype=out)[0].cpu().numpy()
        for b in range(B):
            for f in range(F):
                one = [None if t is None else t[b:b + 1, f:f + 1] for t in (tRs, rn, ry)]
                w1 = P.weights(KINDS[kind], one[0], one[1], one[2], ban=ban, out_dtype=out)[0].cpu().numpy()
                assert np.array_equal(bits(w[b, f]), bits(w1[0, 0])), \
                    (kind, ban, C, b, f, NEIGHBOURS[labels[b, f]], w[b, f], w1[0, 0])


# ----------------------------------------------------------------------------
# exact scaling
# ----------------------------------------------------------------------------
def check_scaling(device, C, F=4, seed=6):
    """Rs * 2^a, Rn * 2^b (a, b in {-40, 0, 40}): PEVD, MVDR, MPDR bit-identical, GEVD scaled by
    exactly 2^(-b/2).  (BAN, rank-1 and the automatic PMWF reference carry an absolute EPSILON
    floor and are checked at a PCM scale by check_eps_floor.)"""
    Rs, Rn, _ = build_batch(seed, C, F, [("cond", 1e6), ("gap", 1e-4), ("pgap", 1e-3)])
    base = {}
    for a in (0, -40, 40):
        for b in (0, -40, 40):
            sRs, sRn = Rs * 2.0 ** a, Rn * 2.0 ** b
            tRs, tRn, tRy = tensors(device, np.complex128, sRs, sRn, sRn)
            got = {
                "pevd": P.weights(_lib.BF_PEVD, tRs)[0],
                "mvdr": P.weights(_lib.BF_MVDR, tRs, tRn)[0],
                "mpdr": P.weights(_lib.BF_MPDR, tRs, None, tRy)[0],
                "gevd": P.weights(_lib.BF_GEVD, tRs, tRn)[0] * 2.0 ** (b // 2),
                "pevd_rn": P.weights(_lib.BF_PEVD, tRs, tRn)[0] * 2.0 ** (b // 2),
            }
            for k, v in got.items():
                v = v.cpu().numpy()
                if (a, b) == (0, 0):
                    base[k] = v
                assert np.array_equal(bits(v), bits(base[k])), (k, C, a, b)


def check_eps_floor(device, C, F=3, seed=7):
    """BAN, rank-1 (gev) and the PMWF automatic reference at a PCM scale (Rn ~ 2^-40), where their
    EPSILON floors bind, against the reference."""
    Rs, Rn, _ = build_batch(seed, C, F, [("cond", 1e2)])
    Rs, Rn = Rs * 2.0 ** -40, Rn * 2.0 ** -40
    tRs, tRn = tensors(device, np.complex128, Rs, Rn)
    refs = [BinRef(Rs[0, f], Rn[0, f]) for f in range(F)]
    w = np.random.default_rng(seed).standard_normal((1, F, C)) + 0j
    out = P.ban(torch.from_numpy(w).to(device), tRn).cpu().numpy()
    for f in range(F):
        d = (np.conj(w[0, f]) @ Rn[0, f] @ w[0, f]).real
        assert d < EPS                                    # the floor binds
        ref, cond = refs[f].ban(w[0, f])
        check(f"setk_ban at the EPSILON floor C={C}", C, out[0, f], ref, cond, False, align=False)
    R1 = P.rank1(tRs, tRn)[0].cpu().numpy()
    for f in range(F):
        ref, cond = refs[f].rank1(True)
        check(f"setk_rank1 gev at the EPSILON floor C={C}", C, R1[0, f].ravel(), ref.ravel(), cond,
              False, align=False)
    w, st, used = P.weights(_lib.BF_PMWF, tRs, tRn, beta=0.0, ref_channel=-1)
    Ws = [r.pmwf_matrix(0.0) for r in refs]
    check_pmwf_ref(Ws, Rn[0], int(used[0]))
    w = w.cpu().numpy()
    for f in range(F):
        W, cond, _ = Ws[f]
        check(f"pmwf auto ref at the EPSILON floor C={C}", C, w[0, f], W[:, int(used[0])], cond,
              False, align=False)
